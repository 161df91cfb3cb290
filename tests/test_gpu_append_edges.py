"""The fused append and attend at the edges a decode loop reaches and continuous synthetic data does not.

* fp16-valued K / V (what the fp16 qkv projection of a decode step hands the append): V tokens then often hold several
  values equal to a threshold.  The fused append's rule for them (kvq_append_kv_fused, DESIGN.md section 2): the V
  outliers are the elements strictly beyond the (n_each+1)-th order statistics, a side left short is padded with
  (0.0, channel 0); K ties at the n_each boundary are taken lowest channel first.  The oracle states the rule as
  OracleCache(v_ties="strict"); the mirror classes keep the reference's topk row.
* engineered K ties (the append's fast tie list and its serial scan) and engineered V vectors (ties, constant and zero
  vectors, values on LUT entries and on midpoints between them);
* other outlier budgets: 3, 41 and 64 per side (64 is the ABI maximum, 128 row entries: the V kernels' tail beyond 64);
* full caches (L == Lmax, Lmax not a multiple of 32): the clamped LUT-row copy, the clamped device-resident length, and
  the device-resident-length append dropping a token that does not fit.

State is compared bit for bit with the oracle (floats by value), attend outputs with the float64 oracle chain at the
suite's tolerances: 1e-3 of the output scale norm-wise, 2e-4 per head (exact tables).  The tests of the oracle's rule
itself run without a GPU."""
import functools

import numpy as np
import pytest
import torch

from _util import O, quantizer, rel_err, spec

DEV = "cuda:0"
gpu = pytest.mark.gpu
THETA = 10000.0


def cu(x):
    return torch.from_numpy(np.ascontiguousarray(x)).to(DEV)


def fp16_tokens(H, L, seed):
    """Synthetic K and V tokens [L, hidden] rounded to fp16 values, as the decode step's fp16 projection yields them."""
    sp = spec(H)
    return (sp.k_tokens(L, seed).astype(np.float16).astype(np.float32),
            sp.v_tokens(L, seed + 1).astype(np.float16).astype(np.float32))


def v_short_sides(v, n_each):
    """Per token: does the upper / lower side hold fewer than n_each values strictly beyond its threshold (a tie)."""
    up, lo = [], []
    for x in np.atleast_2d(v):
        hi, lw, _, _ = O.v_thresholds(x, n_each)
        up.append(int((x > hi).sum()) < n_each)
        lo.append(int((x < lw).sum()) < n_each)
    return np.array(up), np.array(lo)


# ---------------------------------------------------------------------------------------------------------------------
# the oracle's tie rule on hand-built vectors (CPU)
# ---------------------------------------------------------------------------------------------------------------------
def test_strict_v_row_pads_short_sides_and_keeps_order():
    n = 3
    #              0     1    2    3    4    5     6     7    8    9   10    11
    v = np.array([-5.0, 9.0, 7.0, 7.0, 7.0, 0.5, -2.0, -2.0, 1.0, 8.0, -6.0, 0.25], np.float32)
    hi, lo, ui, li = O.v_thresholds(v, n)
    assert (hi, lo) == (7.0, -2.0)        # the 4th largest / smallest; three 7s and two -2s sit on the thresholds
    zp = np.float32(0.5)
    vals, idx = O.v_outlier_row_strict(v, hi, lo, n, zp)
    # upper: 9 (ch 1), 8 (ch 9), one pad; lower: -5 (ch 0), -6 (ch 10), one pad.  Channel 0 entries in the order upper
    # pads, lower outliers, lower pads
    assert idx.tolist() == [0, 0, 0, 1, 9, 10]
    assert vals.tolist() == [0.0, -5.5, 0.0, 8.5, 7.5, -6.5]
    # the reference's row keeps one tied element per short side instead of the pad
    rvals, ridx = O.v_outlier_row(v, ui, li, zp)
    assert sorted(ridx.tolist()) == [0, 1, 2, 6, 9, 10]    # ties lowest index first: channel 2 and channel 6
    assert rvals[ridx.tolist().index(2)] == np.float32(7.0) - zp


def test_strict_v_row_equals_reference_row_without_ties():
    rng = np.random.default_rng(5)
    for _ in range(20):
        v = rng.standard_normal(256).astype(np.float32)
        hi, lo, ui, li = O.v_thresholds(v, 5)
        a = O.v_outlier_row_strict(v, hi, lo, 5, np.float32(0.1))
        b = O.v_outlier_row(v, ui, li, np.float32(0.1))
        assert np.array_equal(a[0], b[0]) and np.array_equal(a[1], b[1])


def test_strict_v_row_constant_and_zero_vectors_are_all_pads():
    for c in (0.0, 0.7, -3.0):
        v = np.full(128, c, np.float32)
        hi, lo, _, _ = O.v_thresholds(v, 4)
        vals, idx = O.v_outlier_row_strict(v, hi, lo, 4, np.float32(c))
        assert hi == lo == np.float32(c) and not vals.any() and not idx.any()


def _one_head_cache(v_ties):
    """H = 1 oracle cache with 3 outliers per side (sparsity 0.96 at hidden 128)."""
    klut, vcent = quantizer(4)
    k1 = {key: (val[:128] if val is not None and key != "cent" else val) for key, val in klut.items()}
    return O.OracleCache(4, 1, 8, k1, vcent, sparsity_threshold=0.96, v_ties=v_ties)


def test_strict_rule_counts_a_tied_element_once():
    """A tied element keeps its nearest dense code under both rules; the reference row adds v - LUT_t[zp] on top of it,
    the strict row does not, so only the strict cache reconstructs the element as its nearest LUT entry."""
    rng = np.random.default_rng(3)
    v = rng.uniform(-1, 1, 128).astype(np.float32)
    v[[10, 20]] = [5.0, 6.0]
    v[[40, 41, 42]] = 3.0            # 3rd to 5th largest: hi = 3, the reference row takes channel 40, the strict one a pad
    k = rng.standard_normal(128).astype(np.float32)
    strict, ref = _one_head_cache("strict"), _one_head_cache("reference")
    assert ref.v_ties == "reference" and O.OracleCache.__init__.__defaults__[-1] == "reference"
    strict.append(k, v)
    ref.append(k, v)
    assert strict.n_each == 3
    assert np.array_equal(strict.vwords, ref.vwords) and np.array_equal(strict.vlut, ref.vlut)
    assert np.array_equal(strict.k_out, ref.k_out) and np.array_equal(strict.k_idx, ref.k_idx)
    lut = strict.vlut[0]
    near = lut[O.nearest_code(v[40:43], np.broadcast_to(lut, (3, lut.size)))]
    assert np.array_equal(strict.v_recon()[40:43, 0], near.astype(np.float64))
    extra = ref.v_recon()[40:43, 0] - near
    zp = lut[O.zero_point_code(4)]
    assert np.count_nonzero(extra) == 1 and extra[0] == np.float32(3.0 - zp)
    # every element strictly beyond a threshold is represented once under both rules
    beyond = (v > 3.0) | (v < np.sort(v)[3])
    assert np.allclose(strict.v_recon()[beyond, 0], v[beyond], atol=1e-6)


def test_k_ties_lowest_channel_first_and_unit_values_zeroed():
    r = np.zeros(16, np.float32)
    r[[3, 5, 9, 12]] = 2.0                                   # upper tie group straddling n_each = 2 + 1
    r[7] = 4.0
    r[[0, 15]] = -1.0                                        # lower group at exactly -1: selected, values zeroed
    lut = np.tile(np.array([-1.0, 1.0], np.float32), (16, 1))
    vals, idx = O.k_outlier_row(r, r, lut, 3)
    assert idx.tolist() == [0, 1, 3, 5, 7, 15]               # 3 and 5 (lowest of the tie), channel 1 (lowest zero)
    assert vals.tolist() == [0.0, 0.0, 1.0, 1.0, 3.0, 0.0]


# ---------------------------------------------------------------------------------------------------------------------
# GPU helpers
# ---------------------------------------------------------------------------------------------------------------------
def fill(bits, H, Lmax, k, v, klut=None, vcent=None, n_dyn=0, n_sink=0, sparsity_threshold=0.99):
    """The same tokens through the strict-rule oracle cache and a LayerCache (the last n_dyn of them through the
    device-resident-length append)."""
    from kvquant_b200.cache import LayerCache
    if klut is None:
        klut, vcent = quantizer(bits, H=H)
    c = O.OracleCache(bits, H, Lmax, klut, vcent, sparsity_threshold=sparsity_threshold, v_ties="strict")
    lc = LayerCache.from_luts(bits, H, Lmax, klut, vcent, device=DEV, n_sink=n_sink,
                              sparsity_threshold=sparsity_threshold)
    kd, vd = cu(k), cu(v)
    L = len(k)
    len_dev = torch.zeros(1, dtype=torch.int64, device=DEV)
    for t in range(L):
        c.append(k[t], v[t])
        if t < L - n_dyn:
            lc.append(kd[t], vd[t])
        else:
            len_dev.fill_(t - 1)
            lc.append_dyn(kd[t], vd[t], len_dev, 1)
    lc.len = L
    return c, lc


def assert_state_matches(lc, c):
    want = dict(kcache=c.kwords, vcache=c.vwords, vlut=c.vlut, vaff=c.vaff, k_outliers=c.k_out,
                k_outlier_idx=c.k_idx, v_outliers=c.v_out, v_outlier_idx=c.v_idx)
    for name, w in want.items():
        got = getattr(lc, name).cpu().numpy()
        tok_axis = 0
        if name.endswith("cache"):
            got, tok_axis = got.reshape(-1, c.Lmax), 1
        if not np.array_equal(got, w):       # (floats by value: +0.0 == -0.0)
            bad = np.nonzero((got != w).any(axis=1 - tok_axis))[0]
            raise AssertionError("%s differs from the oracle at tokens %s" % (name, bad[:12].tolist()))


def check_attend(c, lc, q_seed, sinks=False):
    """Host-length fused attend, native V pass and per-token-LUT V pass, exact tables, against the float64 oracle."""
    H, L, ns = c.H, c.len, lc.n_sink
    q = O.rope_rotate_q(spec(H).q_vec(q_seed), L + ns, THETA)
    s = c.k_scores(q, THETA, ns)
    if sinks:
        g = torch.Generator(device=DEV).manual_seed(q_seed)
        ks = torch.randn((H, 128, ns), generator=g, device=DEV).half()
        vs = torch.randn((H, ns, 128), generator=g, device=DEV).half()
        lc.set_sinks(ks, vs)
        ss = np.einsum("hc,hcn->hn", q.astype(np.float64), ks.cpu().numpy().astype(np.float64))
        p, o = O.attend_ideal(s, c.v_output, sink_scores=ss / np.sqrt(128))
        want = o + np.einsum("hn,hnc->hc", p[:, :ns], vs.cpu().numpy().astype(np.float64))
    else:
        lc.sink_k = lc.sink_v = None
        _, want = O.attend_ideal(s, c.v_output)
    lc.precision = "fp32"
    try:
        for native in (True, False):
            lc.use_native_v = native
            out = lc.attend(cu(q)).cpu().numpy()
            e = rel_err(out, want)[0]
            d = (np.abs(out - want).max(axis=1) / np.abs(want).max(axis=1)).max()
            assert e < 1e-3 and d < 2e-4, (native, sinks, e, d)
    finally:
        lc.use_native_v = True
        lc.sink_k = lc.sink_v = None


def check_legacy_ops(c, lc, seed):
    """The legacy opt2 K and V matvecs on the cache the fused append wrote, against the oracle."""
    import quant_cuda as qc
    H, L, b = c.H, c.len, c.bits
    q = O.rope_rotate_q(spec(H).q_vec(seed), L + 3, THETA)
    mul = torch.zeros((1, H, L), dtype=torch.float32, device=DEV)
    getattr(qc, "vecquant%dmatmul_nuq_perchannel_transposed_rope_mha_batched_fused_opt2" % b)(
        cu(q[None]), lc.kcache, mul, lc.klut.view(H, 128, -1), L, lc.k_outliers, lc.k_outlier_idx, THETA, 3)
    e = rel_err(mul.cpu().numpy()[0], c.k_scores(q, THETA, 3))
    assert e[0] < 1e-4 and e[1] < 1e-4, e
    rng = np.random.default_rng(seed)
    p = O.softmax_f32(rng.standard_normal((H, L)).astype(np.float32) * 3).astype(np.float16).astype(np.float32)
    out = torch.zeros((1, H, 128), dtype=torch.float32, device=DEV)
    getattr(qc, "vecquant%dmatmul_nuq_perchannel_transposed_mha_batched_fused_opt2" % b)(
        cu(p[None]), lc.vcache, out, lc.vlut, L, lc.v_outliers, lc.v_outlier_idx)
    e = rel_err(out.cpu().numpy()[0], c.v_output(p))
    assert e[0] < 1e-4 and e[1] < 1e-4, e


# ---------------------------------------------------------------------------------------------------------------------
# 1-3: fp16-valued tokens
# ---------------------------------------------------------------------------------------------------------------------
FP16_CASES = [(4, 32), (3, 32), (2, 32), (4, 40), (3, 40)]


@functools.lru_cache(maxsize=None)
def fp16_cache(bits, H):
    L = 384 if H == 32 else 320
    k, v = fp16_tokens(H, L, seed=71 if H == 32 else 73)
    c, lc = fill(bits, H, L + 64, k, v, n_dyn=64, n_sink=4)
    return c, lc, k, v


@gpu
@pytest.mark.parametrize("bits,H", FP16_CASES)
def test_fp16_valued_tokens_append_matches_the_strict_oracle(bits, H):
    c, lc, k, v = fp16_cache(bits, H)
    up, lo = v_short_sides(v, c.n_each)
    assert up.sum() >= 8 and lo.sum() >= 8, (up.sum(), lo.sum())     # ties straddling each threshold do occur
    assert_state_matches(lc, c)
    # and they matter: the reference's rule gives other V rows on exactly those tokens
    ref = O.OracleCache(bits, H, c.Lmax, *quantizer(bits, H=H))
    for t in range(len(k)):
        ref.append(k[t], v[t])
    differ = ((ref.v_idx != c.v_idx) | (ref.v_out != c.v_out)).any(axis=1)[:len(k)]
    assert np.array_equal(differ, up | lo)


def _assert_pads_replaced_by_ties(x, n_each, zp, f_vals, f_idx, m_vals, m_idx):
    """The mirror's row == the fused row with each pad replaced by a (distinct) channel whose value equals the
    threshold of that side, its value taken as v - LUT_t[zp]."""
    hi, lo, _, _ = O.v_thresholds(x, n_each)
    n_up, n_lo = int((x > hi).sum()), int((x < lo).sum())
    beyond = (x > hi) | (x < lo)
    fused = sorted(zip(f_idx.tolist(), f_vals.tolist()))
    pads = (n_each - n_up) + (n_each - n_lo)
    for _ in range(pads):
        fused.remove((0, 0.0))
    assert fused == sorted((j, float(np.float32(x[j] - zp))) for j in np.nonzero(beyond)[0])
    assert np.all(np.diff(m_idx) >= 0) and len(set(m_idx.tolist())) == len(m_idx)
    real = [(j, val) for j, val in zip(m_idx.tolist(), m_vals.tolist()) if beyond[j]]
    tied = [(j, val) for j, val in zip(m_idx.tolist(), m_vals.tolist()) if not beyond[j]]
    assert sorted(real) == fused
    assert sum(x[j] == hi for j, _ in tied) == n_each - n_up and sum(x[j] == lo for j, _ in tied) == n_each - n_lo
    assert all(val == float(np.float32(x[j] - zp)) for j, val in tied)


@gpu
@pytest.mark.parametrize("bits", [4, 3])
def test_mirror_classes_keep_the_reference_rule_on_the_same_tokens(bits):
    from kvquant_b200.cache import QuantK, QuantV
    H = 32
    c, lc, k, v = fp16_cache(bits, H)
    L, Lmax, hidden = len(k), c.Lmax, H * 128
    qk = QuantK(bits, hidden, H, max_position_embeddings=Lmax, include_sparse=True)
    qv = QuantV(bits, hidden, H, max_position_embeddings=Lmax, include_sparse=True)
    qk.lookup_table = lc.klut.view(H, 128, -1)
    qk.lookup_table2 = None
    qk.outlier_threshold_lower, qk.outlier_threshold_upper = lc.thr_lower, lc.thr_upper
    qv.lut = lc.v_cent
    q = torch.zeros((H, 1, 128), device=DEV)
    kd, vd = cu(k), cu(v)
    for t in range(L):
        qk.forward_fused_sparse(q, kd[t])
        qv.forward_fused_sparse(torch.full((H, 1, t + 1), 1.0 / (t + 1), device=DEV), vd[t])
    assert torch.equal(qk.kcache, lc.kcache) and torch.equal(qv.vcache, lc.vcache)
    assert torch.equal(qv.lookup_table, lc.vlut)
    assert torch.equal(qk.outliers, lc.k_outliers) and torch.equal(qk.outlier_indices, lc.k_outlier_idx)
    up, lo = v_short_sides(v, c.n_each)
    tie = up | lo
    mv, mi = qv.outliers.cpu().numpy(), qv.outlier_indices.cpu().numpy()
    fv, fi = lc.v_outliers.cpu().numpy(), lc.v_outlier_idx.cpu().numpy()
    assert np.array_equal(mv[:L][~tie], fv[:L][~tie]) and np.array_equal(mi[:L][~tie], fi[:L][~tie])
    zpc = O.zero_point_code(bits)
    for t in np.nonzero(tie)[0]:
        _assert_pads_replaced_by_ties(v[t], c.n_each, c.vlut[t, zpc], fv[t], fi[t], mv[t], mi[t])


@gpu
@pytest.mark.parametrize("sinks", [False, True])
@pytest.mark.parametrize("bits,H", [(4, 32), (3, 32), (2, 32), (4, 40)])
def test_attend_over_an_fp16_built_cache(bits, H, sinks):
    """Pad entries (value 0, channel 0, repeated) go through both V outlier walks."""
    c, lc, _, _ = fp16_cache(bits, H)
    assert (c.v_idx[:c.len] == 0).sum(axis=1).max() >= 2
    check_attend(c, lc, q_seed=bits * 10 + H, sinks=sinks)


# ---------------------------------------------------------------------------------------------------------------------
# 4: engineered K ties
# ---------------------------------------------------------------------------------------------------------------------
def _k_tie_tokens(hidden, n):
    """K tokens under thresholds (-1, 1) on every channel, so the normalised value IS the value.  Each case: tie group
    and how many values lie strictly beyond it, per side; the expected number of group members selected follows."""
    last = hidden - 1
    cases = [  # (upper group, values above it, lower group, values below it)
        (list(range(100, 106)), n - 6, list(range(300, 2300, 250)), n - 8),          # fully selected, fast list
        ([7, 900, 901, 1500, 3000], n - 2, list(range(40, 48)), n - 3),                 # straddling, <= 8 members
        (list(range(1000, 1012)), n - 4, list(range(2, 4000, 133)), n - 10),          # straddling, > 8 members
        ([0, 100, 2000, last], n - 2, [1, 7, last - 1], n - 3),                       # channel 0 / last channel
        ([2, 64, last - 2], n - 3, [0, 9, 4000, last], n - 1),
    ]
    rng = np.random.default_rng(17)
    toks, groups = [], []
    for ug, ua, lg, lb in cases:
        for uval, lval in ((2.5, -2.5), (1.0, -1.0)):           # exactly +-1: selected, value zeroed
            x = rng.uniform(-0.9, 0.9, hidden).astype(np.float32)
            free = np.setdiff1d(np.arange(hidden), ug + lg)
            pick = rng.choice(free, ua + lb, replace=False)
            x[pick[:ua]] = 3.0 + 0.125 * np.arange(ua)
            x[pick[ua:]] = -3.0 - 0.125 * np.arange(lb)
            x[ug] = uval
            x[lg] = lval
            toks.append(x)
            groups.append((ug, min(len(ug), n - ua), lg, min(len(lg), n - lb)))
    return np.stack(toks), groups


@gpu
@pytest.mark.parametrize("bits", [4, 3, 2])
def test_engineered_k_ties(bits):
    H, n = 32, 21
    klut, vcent = quantizer(bits)
    klut = dict(klut, thr_lower=np.full(H * 128, -1.0, np.float32), thr_upper=np.full(H * 128, 1.0, np.float32))
    k, groups = _k_tie_tokens(H * 128, n)
    _, v = fp16_tokens(H, len(k), seed=81)
    c, lc = fill(bits, H, 32, k, v, klut=klut, vcent=vcent, n_dyn=3)
    for t, (ug, nu, lg, nl) in enumerate(groups):    # the construction: lowest channels of each group selected
        row = set(c.k_idx[t].tolist())
        assert [j for j in ug if j in row] == sorted(ug)[:nu] and [j for j in lg if j in row] == sorted(lg)[:nl], t
        if k[t, ug[0]] == 1.0:
            assert not c.k_out[t][np.isin(c.k_idx[t], ug + lg)].any()
    assert_state_matches(lc, c)


# ---------------------------------------------------------------------------------------------------------------------
# 5: engineered V vectors
# ---------------------------------------------------------------------------------------------------------------------
def _v_edge_tokens(hidden, n, vcent):
    rng = np.random.default_rng(23)
    toks = []

    def ties(up_beyond, up_m, lo_beyond, lo_m):
        """Values in (-0.5, 0.5), and per side `beyond` distinct values past m copies of 1.5 / -1.25."""
        x = rng.uniform(-0.5, 0.5, hidden).astype(np.float32)
        ch = rng.permutation(hidden)
        x[ch[:up_beyond]] = 2.0 + 0.0625 * np.arange(1, up_beyond + 1)
        ch = ch[up_beyond:]
        x[ch[:up_m]] = 1.5
        ch = ch[up_m:]
        x[ch[:lo_beyond]] = -2.0 - 0.0625 * np.arange(1, lo_beyond + 1)
        x[ch[lo_beyond:lo_beyond + lo_m]] = -1.25
        return x
    for m in (2, 3, 12):            # ties straddling both thresholds: 1 / 2 / 6 upper pads, 1 / 1 / 6 lower pads
        toks.append(ties(n - (m + 1) // 2, m, n - (1 if m < 12 else 6), m))
    toks.append(ties(n, 3, n, 2))   # values equal to hi / lo but n_each beyond them: no pad
    toks.append(np.full(hidden, 0.7, np.float32))                # constant: hi == lo, sf == 0
    toks.append(np.zeros(hidden, np.float32))                    # all zero
    x = np.zeros(hidden, np.float32)                             # 5 positive entries, the rest 0
    x[rng.choice(hidden, 5, replace=False)] = 1.0 + np.arange(5, dtype=np.float32)
    toks.append(x)
    x = np.zeros(hidden, np.float32)                             # 5 negative entries and a few positive ones
    x[rng.choice(hidden, 5, replace=False)] = -1.0 - np.arange(5, dtype=np.float32)
    x[rng.choice(hidden, 30, replace=False)] = 0.5
    toks.append(x)
    # thresholds exactly -1 / 1 (so LUT_t == the centroids): interior values on LUT entries and on midpoints
    mid = ((vcent[1:] + vcent[:-1]) / np.float32(2)).astype(np.float32)
    inner = np.concatenate([vcent, mid]).astype(np.float32)
    x = np.resize(inner, hidden).astype(np.float32)
    ch = rng.permutation(hidden)[:2 * n + 2]
    x[ch[:n]] = 1.0 + 0.0625 * np.arange(1, n + 1)
    x[ch[n:2 * n]] = -1.0 - 0.0625 * np.arange(1, n + 1)
    x[ch[2 * n]], x[ch[2 * n + 1]] = 1.0, -1.0
    toks.append(x)
    return np.stack(toks).astype(np.float32)


@gpu
@pytest.mark.parametrize("bits", [4, 3, 2])
def test_engineered_v_vectors(bits):
    H, n = 32, 21
    klut, vcent = quantizer(bits)
    v = _v_edge_tokens(H * 128, n, vcent)
    k, _ = fp16_tokens(H, len(v), seed=91)
    c, lc = fill(bits, H, 32, k, v, n_dyn=4)
    up, lo = v_short_sides(v, n)
    assert up[:3].all() and lo[:3].all() and not up[3] and not lo[3]
    assert c.vaff[4, 0] == 0 and c.vaff[5, 0] == 0 and not c.v_idx[4:6].any()
    # the LUT-entry token: its LUT is the centroids, and some midpoints are exact fp32 ties (first entry wins)
    t = len(v) - 1
    assert np.array_equal(c.vlut[t], vcent)
    mid = ((vcent[1:] + vcent[:-1]) / np.float32(2)).astype(np.float32)
    assert (np.abs(vcent[:-1] - mid) == np.abs(vcent[1:] - mid)).any()
    assert_state_matches(lc, c)
    check_attend(c, lc, q_seed=bits)


# ---------------------------------------------------------------------------------------------------------------------
# 6: outlier budgets
# ---------------------------------------------------------------------------------------------------------------------
@gpu
@pytest.mark.parametrize("bits,threshold,n_each", [(4, 0.999, 3), (4, 0.98, 41), (4, 0.969, 64), (3, 0.98, 41),
                                                   (3, 0.969, 64), (2, 0.999, 3)])
def test_outlier_budgets(bits, threshold, n_each):
    H, L = 32, 200
    k, v = fp16_tokens(H, L, seed=101)
    c, lc = fill(bits, H, 256, k, v, n_dyn=16, sparsity_threshold=threshold)
    assert c.n_each == lc.n_each == n_each and lc.n_out == 2 * n_each
    assert_state_matches(lc, c)
    check_attend(c, lc, q_seed=int(threshold * 1000))
    check_legacy_ops(c, lc, seed=n_each)


@gpu
def test_outlier_budget_beyond_the_maximum_is_refused():
    """0.968: 66 per side, 132 row entries > 128.  The append fails with KVQ_E_SHAPE and writes nothing."""
    from kvquant_b200 import _lib
    from kvquant_b200.cache import LayerCache
    klut, vcent = quantizer(4)
    lc = LayerCache.from_luts(4, 32, 64, klut, vcent, device=DEV, sparsity_threshold=0.968)
    assert lc.n_each == 66
    k, v = fp16_tokens(32, 1, seed=5)
    with pytest.raises(_lib.KVQuantError, match=r"\(code -2\)"):
        lc.append(cu(k[0]), cu(v[0]))
    with pytest.raises(_lib.KVQuantError, match=r"\(code -2\)"):
        lc.append_dyn(cu(k[0]), cu(v[0]), torch.zeros(1, dtype=torch.int64, device=DEV))
    torch.cuda.synchronize()
    assert lc.len == 0
    for name in ("kcache", "vcache", "vlut", "vaff", "k_outliers", "k_outlier_idx", "v_outliers", "v_outlier_idx"):
        assert not getattr(lc, name).any(), name


# ---------------------------------------------------------------------------------------------------------------------
# 7: full caches
# ---------------------------------------------------------------------------------------------------------------------
@gpu
@pytest.mark.parametrize("Lmax", [100, 1028])
@pytest.mark.parametrize("bits", [4, 3])
def test_full_cache(bits, Lmax):
    H = 32
    k, v = fp16_tokens(H, Lmax + 1, seed=111)
    c, lc = fill(bits, H, Lmax, k[:Lmax], v[:Lmax], n_dyn=8)
    assert c.len == lc.len == Lmax
    assert_state_matches(lc, c)
    check_attend(c, lc, q_seed=Lmax)
    check_legacy_ops(c, lc, seed=Lmax)
    # device-resident length past the allocation: clamped to Lmax, equal to the host-length attend at L = Lmax
    lc.precision = "fp32"
    q = cu(O.rope_rotate_q(spec(H).q_vec(7), Lmax, THETA))
    want = lc.attend(q).clone()
    len_dev = torch.zeros(1, dtype=torch.int64, device=DEV)
    for ln, add in ((Lmax, 1), (Lmax - 1, 5), (Lmax + 37, 0)):
        len_dev.fill_(ln)
        got = lc.attend_dyn(q, len_dev, add).clone()
        assert rel_err(got.cpu().numpy(), want.cpu().numpy())[0] < 1e-5, (ln, add)
    # the device-resident-length append on a full cache drops the token: nothing changes, slot 0 included
    names = ("kcache", "vcache", "vlut", "vaff", "k_outliers", "k_outlier_idx", "v_outliers", "v_outlier_idx")
    before = {name: getattr(lc, name).clone() for name in names}
    kn, vn = cu(k[Lmax]), cu(v[Lmax])
    for ln, add in ((Lmax, 0), (Lmax - 1, 1), (0, Lmax)):
        len_dev.fill_(ln)
        lc.append_dyn(kn, vn, len_dev, add)
    torch.cuda.synchronize()
    for name in names:
        assert torch.equal(getattr(lc, name), before[name]), name
