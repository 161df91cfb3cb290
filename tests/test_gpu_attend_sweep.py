"""GPU: the decode attend (kvq_attend, kvq_attend_dyn, kvq_attend_merge) and the legacy V / K ops against float64, at
every head count the header accepts (H <= 64, H % 4 == 0), on the kernels' length boundaries and at large positions.

Reference.  Every expected value is computed in float64 from the cache state read back from the device: packed codes
(O.unpack_codes), the K dequantisation table, the outlier rows, and V as v_cent_deq[code] * sf_t + off_t (native form)
or as the per-token LUT rows (LUT form).  cos / sin come from the device RoPE table the attend reads: the oracle's
theta_j may differ from CUDA's powf by one ulp, which at position 70000 moves an angle by ~4e-3 rad and has nothing to do
with the kernels.  The table itself is pinned separately against float64 cos / sin of fl32(theta_j * p).

Two kinds of cache state:
  * realistic: synthetic K / V tokens (fp16-valued) appended with LayerCache.append_chunk;
  * structured probes, written straight into the LayerCache tensors, whose answer is closed-form: a zero K table (every
    score exactly 0: the output is the plain mean of V and the sinks, lse = log(L + n_sink)), or one marked slot per
    head (code 1 against a table whose entry 1 is non-zero, or one K outlier entry) with a scaled score of about 4 at a
    boundary slot.  V holds random packed words, integer centroids, power-of-two scales and integer offsets, so every
    product and sum the V pass forms is exact in fp32.  Each probe asserts that the answer with the marked slot removed,
    moved to a neighbouring slot or rotated one position off differs from the true one by at least 10x the tolerance.

Lengths sit on the kernels' boundaries: 16-token columns, 80-token boxes and 240-token rounds of the exact K kernel,
64-token boxes and 256-token rounds of the fp16-table K kernel, 32-token V tiles, and the lengths (set by the SM count)
where a K range grows from 32 to 64 tokens, a V CTA goes from one tile to two, or every V CTA wraps its stage ring twice.

Tolerances, per head, norm-wise against that head's largest output.  Measured maxima over every case of this module on
an H100 80GB HBM3 (400 W power limit) in brackets:
  * exact tables (fp32), realistic state vs float64, attend and legacy ops: EXACT_TOL = 1.2e-5 (attend 3.6e-6, legacy V
    op 5.0e-7, legacy K op 6.6e-7);
  * lse, |got - want| / max(1, |want|): LSE_TOL = 3e-6 (9.3e-7);
  * probes (exact V sums), exact tables: PROBE_TOL = 4e-6 (1.2e-6);
  * fp16 tables vs the exact-table output on the same state: FP16_TOL = 2e-2 (6.2e-3; per head -- the norm-wise bound
    over all heads in DESIGN section 5 is the looser measure), and FP16_PROBE_TOL = 8e-3 for the marked-slot probes in
    fp16 against float64 (3.9e-3).
Setting KVQ_SWEEP_ERRORS=<path> writes the maxima measured in a run to that JSON file.
"""
import functools
import json
import os
from collections import defaultdict

import numpy as np
import pytest
import torch

from _util import O
from kvquant_b200 import synth

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
THETA = 10000.0
SCALE = 1.0 / np.sqrt(128.0)
HS = tuple(range(4, 65, 4))
FIXED_L = (1, 2, 15, 16, 17, 31, 32, 33, 63, 64, 65, 79, 80, 81, 239, 240, 241, 255, 256, 257)

EXACT_TOL = 1.2e-5
LSE_TOL = 3e-6
PROBE_TOL = 4e-6
FP16_TOL = 2e-2
FP16_PROBE_TOL = 8e-3

MEASURED = defaultdict(float)


@pytest.fixture(scope="module", autouse=True)
def _report_measured():
    yield
    path = os.environ.get("KVQ_SWEEP_ERRORS")
    if path:
        with open(path, "w") as f:
            json.dump(dict(MEASURED), f, indent=1, sort_keys=True)


# ---- shapes the kernels plan from the SM count ------------------------------------------------------------------------
def _sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


def _k_groups(bits, H):          # head groups of the fused K kernels (16 heads per CTA at 4 bits, 32 at 3 / 2 bits)
    return -(-H // (16 if bits == 4 else 32))


def _v_fits(bits, Hg, native):
    """Whether a V CTA of Hg heads gets two ring stages in 227 KB of shared memory: the shared-memory plans of
    launch_vn / vn_smem_layout (kvq_vnative.cu, native form) and launch_v / v_smem_layout (kvq_vaccum.cu, LUT form),
    restated.  The stage of both is the [Hg*W rows x 32 tokens] code slab (the LUT form rounds it up to 32-row boxes)."""
    W, N = 4 * bits, 1 << bits
    if native:   # stages + lane-private pair table + w / w*sf rows (33 / 36-float strides) + 3 mbarriers
        stage = Hg * W * 128
        off_ws = (2 * stage + {4: 256, 3: 64, 2: 16}[bits] * 256 + 2 * Hg * 33 * 4 + 15) // 16 * 16
        total = off_ws + 2 * Hg * 36 * 4 + 8 * 3
    else:        # stages + LUT rows + weights + outlier accumulator + 4 mbarriers
        stage = -(-Hg * W // 32) * 4096
        total = 2 * stage + 2 * 32 * N * 4 + 2 * Hg * 32 * 4 + Hg * 128 * 4 + 8 * 4
    return total + 1024 <= 227 * 1024


def _v_groups(bits, H, native):
    """Head groups of the V pass: 1 while the all-heads slab fits, else 2."""
    return 1 if _v_fits(bits, H, native) else 2


def _sm_lengths(bits, H):
    """The lengths where a K range grows from 32 to 64 tokens and a V CTA goes from one tile to two (and +1)."""
    sms = _sms()
    out = set()
    for n in [32 * max(1, sms // _k_groups(bits, H))] + [32 * max(1, sms // _v_groups(bits, H, nat)) for nat in (True, False)]:
        out |= {n, n + 1}
    return sorted(out)


def _lmax():
    """Pool allocation: >= every SM-derived length, and = 4 (mod 16) so that a full cache's last K and V TMA boxes
    reach past the tensor's last column."""
    return ((32 * _sms() + 2) // 16 + 1) * 16 + 4


def _boundary_slots(bits, H, L):
    """Slots where a kernel's work unit starts or ends: 0, L-1, K ranges, 80-token boxes, 240 / 256-token rounds, 64-token
    boxes, 32-token V tiles and V CTA ranges."""
    sms = _sms()
    R = -(-L // max(1, sms // _k_groups(bits, H)))
    R = (R + 31) // 32 * 32
    s = {0, L - 1}
    for r0 in (0, R, 2 * R):
        for d in (0, 15, 16, 63, 64, 79, 80, 239, 240, 255, 256):
            s |= {r0 + d, r0 + d - 1}
    s |= {R - 1, 2 * R - 1, 31, 32}
    for G in (1, 2):
        n_tiles = -(-L // 32)
        ranges = max(1, sms // G)
        tpc = -(-n_tiles // ranges)
        s |= {32 * tpc - 1, 32 * tpc, 64 * tpc - 1, 64 * tpc}
    return sorted(x for x in s if 0 <= x < L)


# ---- caches ---------------------------------------------------------------------------------------------------------
@functools.lru_cache(maxsize=None)
def _calibration(bits):
    """One calibration at 64 heads; a cache of H heads takes the first H*128 channels."""
    sp = synth.SynthSpec(64, 128, seed=0)
    cal = synth.calibrate(sp, bits, calib_tokens=512, seed=7)
    up, lo, kc = cal["k"]
    return sp, O.build_k_lut(up, lo, kc[0]), np.sort(cal["v"][2][0].ravel().astype(np.float32))


_POOL = {}


def _cache(bits, H, mode="kv", Lmax=None):
    """A pooled LayerCache of (bits, H, outlier mode), emptied and restored to its own tables."""
    from kvquant_b200.cache import LayerCache
    Lmax = Lmax or _lmax()
    key = (bits, H, mode, Lmax)
    lc = _POOL.get(key)
    if lc is None:
        sp, klut, vcent = _calibration(bits)
        n = H * 128
        kl = dict(lut=klut["lut"][:n], thr_lower=klut["thr_lower"][:n], thr_upper=klut["thr_upper"][:n])
        lc = LayerCache.from_luts(bits, H, Lmax, kl, vcent, device=DEV, include_sparse=mode != "dense",
                                  sparse_v=mode == "kv")
        lc._own_tables = (lc.klut_deq, lc.v_cent_deq)
        _POOL[key] = lc
    lc.reset()
    lc.klut_deq, lc.v_cent_deq = lc._own_tables
    lc.n_sink, lc.pos_base, lc.sink_k, lc.sink_v = 0, 0, None, None
    lc.use_native_v, lc.precision = True, "fp32"
    return lc


def _tokens(lc, T, seed):
    """T synthetic fp16-valued K / V tokens [T, hidden] on the device (the synth distributions)."""
    sp = _calibration(lc.bits)[0]
    n = lc.hidden
    g = torch.Generator(device=DEV).manual_seed(seed)
    mu = torch.as_tensor(sp.mu[:n], device=DEV)
    sigma = torch.as_tensor(sp.sigma[:n], device=DEV)
    k = torch.randn((T, n), generator=g, device=DEV) * sigma + mu
    k = k + (torch.rand((T, n), generator=g, device=DEV) < 0.005) * torch.randn((T, n), generator=g, device=DEV) * 6 * sigma
    st = torch.exp(torch.randn((T, 1), generator=g, device=DEV) * 0.3)
    v = torch.randn((T, n), generator=g, device=DEV) * st
    v = v + (torch.rand((T, n), generator=g, device=DEV) < 0.005) * torch.randn((T, n), generator=g, device=DEV) * 6 * st
    return k.half().float().contiguous(), v.half().float().contiguous()


def _fill(lc, L, seed=0):
    k, v = _tokens(lc, L, seed)
    lc.append_chunk(k, v)
    return lc


def _sinks(lc, n, seed, zero_k=False, int_v=False):
    lc.n_sink = n
    g = torch.Generator(device=DEV).manual_seed(seed)
    if zero_k:
        ks = torch.zeros((lc.H, 128, n), device=DEV)
    else:
        ks = torch.randn((lc.H, 128, n), generator=g, device=DEV)
    if int_v:
        vs = torch.randint(-4, 5, (lc.H, n, 128), generator=g, device=DEV).float()
    else:
        vs = torch.randn((lc.H, n, 128), generator=g, device=DEV)
    lc.set_sinks(ks.half(), vs.half())


def _query(H, seed, kind="random"):
    rng = np.random.default_rng([seed, H])
    q = rng.standard_normal((H, 128)).astype(np.float16).astype(np.float32)
    if kind == "zeros":   # exact zeros: single channels, a whole rotary pair (c, c^64) and a whole head
        q[:, 5] = 0.0
        q[:, 70] = 0.0
        q[:, 9] = q[:, 9 + 64] = 0.0
        q[H // 2] = 0.0
    elif kind == "tiny":  # channels of ~1e-20 next to O(1) rotary partners
        q[:, 3] = 1e-20
        q[:, 64 + 17] = -3e-20
    return q


def cu(x):
    return torch.from_numpy(np.ascontiguousarray(x)).to(DEV)


# ---- float64 reference from the device state --------------------------------------------------------------------------
def _rope(lc, p0, L):
    from kvquant_b200 import quant_cuda as qc
    rope, _, _ = qc.rope_tables(lc.device, THETA, p0 + L + 1)
    cs = rope[:, p0:p0 + L].double().cpu().numpy()           # [64, L, 2]
    return np.concatenate([cs[..., 0]] * 2), np.concatenate([cs[..., 1]] * 2)   # [128, L]: channel c -> pair c % 64


def _raw_scores(lc, L, q, pos_offset):
    """q.K^T, unscaled, float64 [H, L]: dense codes through klut_deq plus the K outlier entries, rotated with the device
    table at positions t + pos_offset."""
    H, bits = lc.H, lc.bits
    q = np.asarray(q, dtype=np.float64).reshape(H, 128)
    s = np.zeros((H, L))
    if L == 0:
        return s
    cos, sin = _rope(lc, pos_offset, L)
    sign = np.where(np.arange(128) < 64, 1.0, -1.0)
    partner = (np.arange(128) + 64) % 128
    codes = O.unpack_codes(lc.kcache[:, :, :L].cpu().numpy().reshape(H * 4 * bits, L), bits).astype(np.int64)
    lut = lc.klut_deq.double().cpu().numpy()
    for h in range(H):
        sl = slice(h * 128, (h + 1) * 128)
        K = np.take_along_axis(lut[sl], codes[sl], axis=1)
        s[h] = (K * (q[h][:, None] * cos + (sign * q[h][partner])[:, None] * sin)).sum(0)
    if lc.sparse_k:
        val = lc.k_outliers[:L].double().cpu().numpy()
        idx = lc.k_outlier_idx[:L].cpu().numpy().astype(np.int64)
        t = np.broadcast_to(np.arange(L)[:, None], idx.shape)
        head, ch = idx // 128, idx % 128
        qf = q.ravel()
        contrib = val * (cos[ch, t] * qf[idx] + np.where(ch < 64, 1.0, -1.0) * sin[ch, t] * qf[head * 128 + partner[ch]])
        np.add.at(s, (head, t), contrib)
    return s


def _v_sum(lc, L, w, native=True):
    """sum_t w[h, t] * V[h, :, t] in float64 [H, 128], V from the native (v_cent_deq, vaff) or the LUT-row form."""
    H, bits = lc.H, lc.bits
    out = np.zeros((H, 128))
    if L == 0:
        return out
    codes = O.unpack_codes(lc.vcache[:, :, :L].cpu().numpy().reshape(H * 4 * bits, L), bits).astype(np.int64)
    if native:
        cent = lc.v_cent_deq.double().cpu().numpy()
        aff = lc.vaff[:L].double().cpu().numpy()
    else:
        vlut = lc.vlut[:L].double().cpu().numpy()
    for h in range(H):
        c = codes[h * 128:(h + 1) * 128]
        V = cent[c] * aff[:, 0] + aff[:, 1] if native else vlut[np.arange(L)[None, :], c]
        out[h] = V @ w[h]
    if lc.sparse_v:
        val = lc.v_outliers[:L].double().cpu().numpy()
        idx = lc.v_outlier_idx[:L].cpu().numpy().astype(np.int64)
        t = np.broadcast_to(np.arange(L)[:, None], idx.shape)
        flat = out.ravel()
        np.add.at(flat, idx, val * w[idx // 128, t])
        out = flat.reshape(H, 128)
    return out


def _v_slot(lc, t, native=True):
    """V of slot t, float64 [H, 128] (dequantised value plus its outlier entries)."""
    H, bits = lc.H, lc.bits
    c = O.unpack_codes(lc.vcache[:, :, t].cpu().numpy().reshape(H * 4 * bits, 1), bits)[:, 0].astype(np.int64)
    if native:
        sf, off = lc.vaff[t].double().cpu().numpy()
        V = lc.v_cent_deq.double().cpu().numpy()[c] * sf + off
    else:
        V = lc.vlut[t].double().cpu().numpy()[c]
    if lc.sparse_v:
        np.add.at(V, lc.v_outlier_idx[t].cpu().numpy().astype(np.int64), lc.v_outliers[t].double().cpu().numpy())
    return V.reshape(H, 128)


def _softmax_out(lc, s_scaled, q, native=True, sink_scores=None):
    """Attention output and lse from float64 scaled scores [H, L] plus the cache's sinks (their scaled scores computed
    from q and sink_k, or given as sink_scores [H, n_sink])."""
    H, L = s_scaled.shape
    m = s_scaled.max(axis=1) if L else np.full(H, -np.inf)
    ns = lc.n_sink if lc.sink_k is not None else 0
    if ns:
        sk = lc.sink_k.double().cpu().numpy()
        sv = lc.sink_v.double().cpu().numpy()
        ss = SCALE * np.einsum("hc,hci->hi", np.asarray(q, dtype=np.float64).reshape(H, 128), sk)
        if sink_scores is not None:
            ss = sink_scores
        m = np.maximum(m, ss.max(axis=1))
    e = np.exp(s_scaled - m[:, None])
    l = e.sum(axis=1)
    o = _v_sum(lc, L, e, native)
    if ns:
        es = np.exp(ss - m[:, None])
        l = l + es.sum(axis=1)
        o = o + np.einsum("hi,hic->hc", es, sv)
    return o / l[:, None], m + np.log(l)


def _reference(lc, q, native=True):
    L = lc.len
    return _softmax_out(lc, SCALE * _raw_scores(lc, L, q, lc.n_sink + lc.pos_base), q, native)


# ---- comparisons ------------------------------------------------------------------------------------------------------
def _head_err(got, want):
    got, want = np.asarray(got, dtype=np.float64), np.asarray(want, dtype=np.float64)
    return (np.abs(got - want).max(axis=1) / np.maximum(np.abs(want).max(axis=1), 1e-30)).max()


def _check(cat, got, want, tol, what=""):
    e = float(_head_err(got, want))
    MEASURED[cat] = max(MEASURED[cat], e)
    assert np.isfinite(got).all() and e <= tol, (cat, what, e, tol)


def _check_lse(got, want, what=""):
    got, want = np.asarray(got, dtype=np.float64), np.asarray(want, dtype=np.float64)
    e = float((np.abs(got - want) / np.maximum(1.0, np.abs(want))).max())
    MEASURED["lse"] = max(MEASURED["lse"], e)
    assert np.isfinite(got).all() and e <= LSE_TOL, ("lse", what, e)


def _run(lc, q, precision="fp32", native=True, dyn=None, L_cap=None):
    """(out, lse) of kvq_attend, or of kvq_attend_dyn with dyn = (len_dev value, len_add)."""
    lc.precision, lc.use_native_v = precision, native
    qd = cu(q)
    lse = torch.full((lc.H,), float("nan"), device=DEV)
    out = torch.full((lc.H, 128), float("nan"), device=DEV)
    if dyn is None:
        lc.attend(qd, out=out, lse=lse)
    else:
        len_dev = torch.full((1,), dyn[0], dtype=torch.int64, device=DEV)
        lc.attend_dyn(qd, len_dev, dyn[1], out=out, lse=lse, L_cap=L_cap)
    torch.cuda.synchronize()
    return out.cpu().numpy().astype(np.float64), lse.cpu().numpy().astype(np.float64)


def _check_all_forms(lc, q, what, dyn=True):
    """Exact tables in the native and LUT V forms and (native) the device-resident length against float64; the fp16
    tables against the exact-table output on the same state."""
    want_o, want_l = _reference(lc, q, native=True)
    o, l = _run(lc, q)
    _check("exact", o, want_o, EXACT_TOL, what)
    _check_lse(l, want_l, what)
    if dyn and lc.len > 0:
        for v, add in ((lc.len, 0), (lc.len - 1, 1)):
            od, ld = _run(lc, q, dyn=(v, add))
            _check("exact", od, want_o, EXACT_TOL, what + " dyn")
            _check_lse(ld, want_l, what + " dyn")
    o16, _ = _run(lc, q, precision="fp16")
    _check("fp16_vs_exact", o16, o, FP16_TOL, what + " fp16")
    if lc.v_norm is None:
        lut_o, lut_l = _reference(lc, q, native=False)
        ol, ll = _run(lc, q, native=False)
        _check("exact", ol, lut_o, EXACT_TOL, what + " lut")
        _check_lse(ll, lut_l, what + " lut")


# ---- the RoPE table -----------------------------------------------------------------------------------------------
def test_rope_table_matches_float64_up_to_past_2_18():
    """Each entry against float64 cos / sin of fl32(theta_j * p), allowing theta_j one ulp off the float64 pow; the fp16
    table is the fp32 one rounded to fp16."""
    from kvquant_b200 import quant_cuda as qc
    npos_min = (1 << 18) + 300
    rope, rope_h, npos = qc.rope_tables(torch.device(DEV), THETA, npos_min)
    rng = np.random.default_rng(0)
    pos = np.unique(np.concatenate([np.arange(0, 4096), np.arange(65536 - 64, 65536 + 64),
                                    np.arange((1 << 18) - 64, (1 << 18) + 256), rng.integers(0, npos_min, 4096)]))
    pi = torch.as_tensor(pos, device=DEV)
    tab = rope[:, pi].double().cpu().numpy()                                  # [64, P, 2]
    th = O.rope_theta_vec(THETA)[:64].astype(np.float32)
    arg = (th[:, None] * pos.astype(np.float32)[None, :]).astype(np.float32)
    bound = (pos[None, :] * np.spacing(th)[:, None].astype(np.float64) + 1.01 * np.spacing(np.abs(arg)).astype(np.float64)
             + 4e-7)
    for k, fn in ((0, np.cos), (1, np.sin)):
        d = np.abs(tab[..., k] - fn(arg.astype(np.float64)))
        assert (d <= bound).all(), (k, d.max(), np.unravel_index(np.argmax(d - bound), d.shape))
    # the pair j = 0 has theta exactly 1: only the argument's own rounding and cosf / sinf remain
    assert np.abs(tab[0, :, 0] - np.cos(pos.astype(np.float32).astype(np.float64))).max() < 5e-7
    half = rope_h[:, pi].cpu().numpy().view(np.float16).reshape(64, len(pos), 2).astype(np.float64)
    assert np.array_equal(half, tab.astype(np.float32).astype(np.float16).astype(np.float64))


# ---- realistic sweep ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("H", HS)
@pytest.mark.parametrize("bits", (4, 3, 2))
def test_attend_every_head_count(bits, H):
    """Every (bits, H), both table precisions, native and LUT V forms, host and device length, out and lse, at a
    length past an exact-K round and one past an fp16-K round and a V tile, with 3 sinks."""
    lc = _fill(_cache(bits, H), 257, seed=H)
    _sinks(lc, 3, seed=bits * 100 + H)
    for L in (241, 257):
        lc.len = L
        _check_all_forms(lc, _query(H, L), "bits=%d H=%d L=%d" % (bits, H, L))


@pytest.mark.parametrize("L", [0, 1, 300])
@pytest.mark.parametrize("bits,H", [(4, 4), (4, 48), (3, 36), (3, 64), (2, 28)])
def test_attend_64_sinks_with_distinct_scores(bits, H, L):
    """n_sink = 64 (the maximum) with random fp16 sink keys: every (head, sink) pair has its own score, so a sink-score
    row stride below 64 (rows of neighbouring heads overlapping) changes the result.  L = 0 is the sinks-only call."""
    lc = _fill(_cache(bits, H), max(L, 1), seed=17)
    lc.len = L
    _sinks(lc, 64, seed=bits * 1000 + H)
    q = _query(H, 64 + L) * 0.25      # token scores of a few units, which the sinks below can lead
    # make each head's leading sink one of its first 32 (the sinks a shorter row stride would overwrite) and scale the
    # head's sink keys (by at most 8: a score of magnitude |s| carries an fp32 rounding of |s| * 6e-8) so that it leads
    # the token scores by 1
    s = SCALE * _raw_scores(lc, L, q, lc.n_sink) if L else np.full((H, 1), -np.inf)
    sk, sv = lc.sink_k.clone(), lc.sink_v.clone()
    ss = SCALE * np.einsum("hc,hci->hi", q.astype(np.float64), sk.double().cpu().numpy())
    for h in np.nonzero(ss.argmax(axis=1) >= 32)[0]:
        sk[h] = torch.cat([sk[h, :, 32:], sk[h, :, :32]], dim=1)
        sv[h] = torch.cat([sv[h, 32:], sv[h, :32]], dim=0)
        ss[h] = np.concatenate([ss[h, 32:], ss[h, :32]])
    a = np.clip((s.max(axis=1) + 1.0) / ss[:, :32].max(axis=1), 1.0, 8.0)
    lc.set_sinks((sk.float() * torch.as_tensor(a, device=DEV).float()[:, None, None]).half(), sv)
    want_o, _ = _reference(lc, q)
    # sensitivity: sink-score rows 32 floats apart (head h >= 1 reading sinks 32..63 of head h-1 as its first 32) give
    # answers far outside the tolerance
    ss = SCALE * np.einsum("hc,hci->hi", q.astype(np.float64), lc.sink_k.double().cpu().numpy())
    ss_alt = ss.copy()
    ss_alt[1:, :32] = ss[:-1, 32:]
    alt, _ = _softmax_out(lc, SCALE * _raw_scores(lc, L, q, lc.n_sink), q, sink_scores=ss_alt)
    assert (_alt_err(want_o, [alt])[1:] >= 10 * EXACT_TOL).all()
    _check_all_forms(lc, q, "64 sinks bits=%d H=%d L=%d" % (bits, H, L))


@pytest.mark.parametrize("mode", ["kv", "k_only", "dense"])
@pytest.mark.parametrize("bits,H", [(4, 44), (3, 52), (2, 20), (4, 64)])
def test_attend_outlier_modes(bits, H, mode):
    lc = _fill(_cache(bits, H, mode), 600, seed=7)
    for L in (33, 600):
        lc.len = L
        _check_all_forms(lc, _query(H, 1 + L), "%s bits=%d H=%d L=%d" % (mode, bits, H, L))


@pytest.mark.parametrize("H", (4, 32, 52, 64))
@pytest.mark.parametrize("bits", (4, 3, 2))
def test_attend_every_boundary_length(bits, H):
    """The fixed boundary lengths, the SM-derived ones and a full cache (Lmax = 4 mod 16: the last K and V boxes reach
    past the tensor)."""
    lc = _cache(bits, H)
    Lmax = lc.Lmax
    _fill(lc, Lmax, seed=1)
    q = _query(H, 5)
    for L in sorted(set(FIXED_L) | set(_sm_lengths(bits, H)) | {Lmax}):
        lc.len = L
        want_o, want_l = _reference(lc, q)
        o, l = _run(lc, q)
        _check("exact", o, want_o, EXACT_TOL, "L=%d" % L)
        _check_lse(l, want_l, "L=%d" % L)
        o16, _ = _run(lc, q, precision="fp16")
        _check("fp16_vs_exact", o16, o, FP16_TOL, "fp16 L=%d" % L)
        if L in (1, 80, 257, Lmax):
            lut_o, _ = _reference(lc, q, native=False)
            _check("exact", _run(lc, q, native=False)[0], lut_o, EXACT_TOL, "lut L=%d" % L)


@pytest.mark.parametrize("pos_end", [1234, 65536, 65537, (1 << 18) + 77])
@pytest.mark.parametrize("bits,H", [(4, 32), (3, 52), (2, 64)])
def test_attend_at_large_positions(bits, H, pos_end):
    """pos_base so that L + n_sink + pos_base = pos_end: 65536 still gathers the outlier cos / sin from the table,
    65537 takes the outlier scatter's direct cos / sin branch."""
    L = 300
    lc = _fill(_cache(bits, H), L, seed=3)
    _sinks(lc, 2, seed=4)
    lc.pos_base = pos_end - L - 2
    _check_all_forms(lc, _query(H, pos_end), "pos_end=%d" % pos_end)


@pytest.mark.parametrize("kind", ["zeros", "tiny"])
@pytest.mark.parametrize("bits,H", [(4, 40), (3, 12), (2, 64)])
def test_attend_queries_with_zero_and_tiny_channels(bits, H, kind):
    """Exact zeros (single channels, a whole rotary pair, a whole head) and ~1e-20 channels next to O(1) partners: the
    exact K form divides by q_c and substitutes 1e-30 for an exact zero."""
    lc = _fill(_cache(bits, H), 400, seed=5)
    q = _query(H, 9, kind)
    _check_all_forms(lc, q, kind)
    if kind == "zeros":
        o, _ = _run(lc, q)
        assert np.isfinite(o).all()


# ---- device-resident length ---------------------------------------------------------------------------------------
@pytest.mark.parametrize("bits,H", [(4, 36), (3, 60), (2, 8)])
def test_attend_dyn_clamps_and_caps(bits, H):
    """len_dev + len_add past L_cap clamps to L_cap; L_cap < Lmax; several lengths under one cap."""
    lc = _fill(_cache(bits, H), 700, seed=6)
    q = _query(H, 2)
    L_cap = 500
    for L, dyn in ((500, (900, 0)), (500, (499, 1)), (321, (320, 1)), (1, (0, 1))):
        lc.len = L
        want_o, want_l = _reference(lc, q)
        for prec in ("fp32", "fp16"):
            o, l = _run(lc, q, precision=prec, dyn=dyn, L_cap=L_cap)
            if prec == "fp32":
                _check("exact", o, want_o, EXACT_TOL, "dyn L=%d" % L)
                _check_lse(l, want_l)
            else:
                _check("fp16_vs_exact", o, _run(lc, q, dyn=dyn, L_cap=L_cap)[0], FP16_TOL, "dyn fp16 L=%d" % L)


# ---- sequence-sharded merge ---------------------------------------------------------------------------------------
@pytest.mark.parametrize("cuts", [(0, 417, 1000), (0, 1, 260, 1000), (0, 333, 334, 701, 1000)])
@pytest.mark.parametrize("bits,H", [(4, 48), (3, 28)])
def test_attend_merge_of_shards_equals_full_attention(bits, H, cuts):
    """Shards cut off the 32-token grid (one of them a single token), sinks on shard 0 only, each shard at its own
    pos_base; kvq_attend_merge of the shards' (out, lse) against the float64 attention over the whole sequence."""
    from kvquant_b200 import _lib
    from kvquant_b200.cache import LayerCache
    n_sink, T = 4, cuts[-1]
    base = _cache(bits, H)
    k, v = _tokens(base, T, seed=11)
    q = _query(H, 3)
    parts, scores, shards = [], [], []
    for r in range(len(cuts) - 1):
        a, b = cuts[r], cuts[r + 1]
        lc = LayerCache(bits, H, (b - a + 15) // 16 * 16 + 16, base.klut, None, base.thr_lower, base.thr_upper,
                        base.v_cent, DEV, n_sink=n_sink if r == 0 else 0)
        if r == 0:
            g = torch.Generator(device=DEV).manual_seed(12)
            lc.set_sinks(torch.randn((H, 128, n_sink), generator=g, device=DEV).half(),
                         torch.randn((H, n_sink, 128), generator=g, device=DEV).half())
        else:
            lc.pos_base = n_sink + a
        lc.append_chunk(k[a:b].contiguous(), v[a:b].contiguous())
        o, l = _run(lc, q)
        parts.append(np.concatenate([o.ravel(), l]))
        scores.append(SCALE * _raw_scores(lc, b - a, q, lc.n_sink + lc.pos_base))
        shards.append(lc)
    pd = cu(np.stack(parts).astype(np.float32))
    out = torch.empty((H, 128), device=DEV)
    lib = _lib.load()
    _lib.check(lib.kvq_attend_merge(pd.data_ptr(), len(parts), H, out.data_ptr(), torch.cuda.current_stream().cuda_stream))
    # float64 attention over sinks + every shard's tokens
    s = np.concatenate(scores, axis=1)
    sk, sv = shards[0].sink_k.double().cpu().numpy(), shards[0].sink_v.double().cpu().numpy()
    ss = SCALE * np.einsum("hc,hci->hi", q.astype(np.float64), sk)
    m = np.maximum(s.max(axis=1), ss.max(axis=1))
    o_num = np.einsum("hi,hic->hc", np.exp(ss - m[:, None]), sv)
    l = np.exp(ss - m[:, None]).sum(axis=1)
    for lc, sc in zip(shards, scores):
        e = np.exp(sc - m[:, None])
        o_num += _v_sum(lc, sc.shape[1], e)
        l += e.sum(axis=1)
    _check("exact", out.cpu().numpy(), o_num / l[:, None], EXACT_TOL, "merge %s" % (cuts,))


# ---- structured probes ----------------------------------------------------------------------------------------------
def _rand_words(shape, g):
    lo = torch.randint(0, 1 << 16, shape, generator=g, device=DEV, dtype=torch.int64)
    hi = torch.randint(0, 1 << 16, shape, generator=g, device=DEV, dtype=torch.int64)
    w = (hi << 16) | lo
    return torch.where(w >= (1 << 31), w - (1 << 32), w).to(torch.int32)


def _probe_v(lc, L, seed, v_out=True):
    """Random packed V words, integer centroids, power-of-two scales and integer offsets (LUT rows to match), and
    optionally integer V outlier entries: every product and sum of the V pass is exact in fp32."""
    H, N = lc.H, 1 << lc.bits
    g = torch.Generator(device=DEV).manual_seed(seed)
    lc.vcache[:, :, :L] = _rand_words((H, 4 * lc.bits, L), g)
    lc.v_cent_deq = (torch.arange(N, device=DEV, dtype=torch.float32) - N // 2).contiguous()
    sf = torch.tensor([0.5, 1.0, 2.0], device=DEV)[torch.randint(0, 3, (L,), generator=g, device=DEV)]
    off = torch.randint(-4, 5, (L,), generator=g, device=DEV).float()
    lc.vaff[:L, 0], lc.vaff[:L, 1] = sf, off
    lc.vlut[:L] = lc.v_cent_deq[None, :] * sf[:, None] + off[:, None]
    if lc.sparse_v:
        if v_out:
            idx = torch.randint(0, lc.hidden, (L, lc.n_out), generator=g, device=DEV).sort(dim=1).values
            lc.v_outlier_idx[:L] = idx.int()
            lc.v_outliers[:L] = torch.randint(-3, 4, (L, lc.n_out), generator=g, device=DEV).float()
        else:
            lc.v_outliers[:L] = 0.0


def _probe_k_zero(lc, L, seed):
    """Random K codes against an all-zero table and no K outlier entries: every score is exactly 0."""
    g = torch.Generator(device=DEV).manual_seed(seed)
    lc.kcache[:, :, :L] = _rand_words((lc.H, 4 * lc.bits, L), g)
    lc.klut_deq = torch.zeros_like(lc._own_tables[0])
    if lc.sparse_k:
        lc.k_outliers[:L] = 0.0
        lc.k_outlier_idx[:L] = 0


def _alt_err(want, alts):
    """Per head: the smallest norm-wise distance of an alternative answer from the true one."""
    want = np.asarray(want)
    d = np.full(want.shape[0], np.inf)
    for a in alts:
        d = np.minimum(d, np.abs(a - want).max(axis=1) / np.abs(want).max(axis=1))
    return d


def _coverage_case(bits, H, L, n_sink, native, precision, dyn, v_out, Lmax=None):
    lc = _cache(bits, H, Lmax=Lmax)
    _probe_k_zero(lc, L, seed=L)
    _probe_v(lc, L, seed=L + 1, v_out=v_out)
    lc.len = L
    if n_sink:
        _sinks(lc, n_sink, seed=n_sink, zero_k=True, int_v=True)
    q = _query(H, 1)
    w = np.ones((H, L))
    num = _v_sum(lc, L, w, native)
    sv = lc.sink_v.double().cpu().numpy().sum(axis=1) if n_sink else 0.0
    n = L + n_sink
    want = (num + sv) / n
    # sensitivity: slot 0, slot L-1 or a sink dropped, or slot 0 counted twice
    alts = []
    if L:
        V0, Vl = _v_slot(lc, 0, native), _v_slot(lc, L - 1, native)
        alts += [(num + sv - V0) / (n - 1) if n > 1 else np.zeros_like(want), (num + sv - Vl) / max(n - 1, 1),
                 (num + sv + V0) / (n + 1)]
    if n_sink and n > 1:
        alts.append((num + sv - lc.sink_v.double().cpu().numpy()[:, 0]) / (n - 1))
    tol = PROBE_TOL
    assert (_alt_err(want, alts) >= 10 * tol).all()
    o, l = _run(lc, q, precision=precision, native=native, dyn=(L, 0) if dyn else None)
    _check("probe", o, want, tol, "coverage bits=%d H=%d L=%d" % (bits, H, L))
    _check_lse(l, np.full(H, np.log(n)), "coverage L=%d" % L)
    assert np.abs(l - np.log(n)).max() < 0.1 / n     # an off-by-one count moves lse by 1/n


@pytest.mark.parametrize("L", list(FIXED_L) + ["sm"])
@pytest.mark.parametrize("bits,H", [(4, 4), (4, 44), (3, 36), (3, 60), (2, 52)])
def test_coverage_probe_every_slot_once(bits, H, L):
    """Zero K table: the output is the plain mean of V and the sinks, lse = log(L + n_sink).  Native and LUT V forms,
    both precisions, host and device length."""
    Ls = _sm_lengths(bits, H) if L == "sm" else [L]
    for L in Ls:
        for native, precision, dyn in ((True, "fp32", False), (True, "fp16", True), (False, "fp32", False)):
            _coverage_case(bits, H, L, 1 if L % 2 else 0, native, precision, dyn, v_out=L % 3 != 0)


@pytest.mark.parametrize("n_sink,L", [(64, 0), (1, 0), (64, 1), (64, 300)])
@pytest.mark.parametrize("bits,H", [(4, 64), (3, 4), (2, 32)])
def test_coverage_probe_sinks(bits, H, n_sink, L):
    """n_sink = 64 (the maximum) and 1, with L = 0 (sinks only) and with tokens."""
    for native in (True, False):
        _coverage_case(bits, H, L, n_sink, native, "fp32", False, v_out=True)


@pytest.mark.parametrize("bits,H,native", [(4, 32, True), (4, 48, False), (3, 52, False), (2, 64, True)])
def test_coverage_probe_ring_wraps_twice(bits, H, native):
    """A length where every V CTA streams at least 9 tiles (a 4-stage ring wrapped twice), beyond what the float64 host
    reference would take: the closed-form probe."""
    G = _v_groups(bits, H, native)
    L = 32 * 9 * max(1, _sms() // G) + 17
    Lmax = (L + 15) // 16 * 16 + 4
    _coverage_case(bits, H, L, 3, native, "fp32", native, v_out=True, Lmax=Lmax)


def _marked_case(bits, H, L, form, pos_base, precision, native=True, n_sink=0):
    """One marked slot per head at boundary slots; all other scores exactly 0."""
    lc = _cache(bits, H)
    _probe_k_zero(lc, L, seed=L + 5)
    lc.kcache[:, :, :L] = 0
    _probe_v(lc, L, seed=L + 6, v_out=True)
    lc.len = L
    lc.pos_base = pos_base
    if n_sink:
        _sinks(lc, n_sink, seed=3, zero_k=True, int_v=True)
    p0 = lc.n_sink + pos_base
    slots = _boundary_slots(bits, H, L)
    s_h = np.array([slots[(h * 7) % len(slots)] for h in range(H)])
    q = _query(H, 21).astype(np.float64)
    partner = (np.arange(128) + 64) % 128
    sign = np.where(np.arange(128) < 64, 1.0, -1.0)
    cos, sin = _rope(lc, p0, L + 1)
    small = np.r_[0:4, 64:68]                                            # pairs j < 4: theta_j >= 0.65 rad per position

    def rq(h, t):     # the rotated query of head h at slot t (channels 0..127)
        return q[h] * cos[:, t] + sign * q[h][partner] * sin[:, t]
    lut = torch.zeros_like(lc._own_tables[0]).cpu()
    mark = {}         # outlier form: head -> (channel, value)
    for h in range(H):
        r = rq(h, s_h[h])
        if form == "dense":   # u along the rotated query: one position later every pair has turned by >= 0.65 rad,
            u = np.zeros(128)  # so the score drops from 5 to at most 5 cos(0.65) < 4
            u[small] = r[small]
            u *= 5.0 / (SCALE * (u * r).sum())
            u = u.astype(np.float32).astype(np.float64)
            lut[h * 128:(h + 1) * 128, 1] = torch.from_numpy(u).float()
            words = O.pack_codes(np.ones((128, 1), dtype=np.uint8), bits)[:, 0]
            lc.kcache[h, :, s_h[h]] = torch.from_numpy(words.astype(np.int32)).to(DEV)
        else:
            r1 = rq(h, s_h[h] + 1)
            c = int(small[np.argmax(np.minimum(np.abs(r[small]), np.abs(r[small] - r1[small])))])
            val = np.float32(5.0 / (SCALE * r[c]))
            mark[h] = (c, float(val))
            k = int((lc.k_outliers[s_h[h]] != 0).sum().item())
            lc.k_outliers[s_h[h], lc.n_out - 1 - k] = float(val)
            lc.k_outlier_idx[s_h[h], lc.n_out - 1 - k] = h * 128 + c
    if form == "outlier":   # rows sorted by channel, (0.0, channel 0) pads in front
        for t in set(s_h.tolist()):
            order = lc.k_outlier_idx[t].long().argsort()
            lc.k_outlier_idx[t] = lc.k_outlier_idx[t][order].clone()
            lc.k_outliers[t] = lc.k_outliers[t][order].clone()
    lc.klut_deq = lut.to(DEV).contiguous()
    s = SCALE * _raw_scores(lc, L, q, p0)
    want, want_l = _softmax_out(lc, s, q, native)
    assert (np.abs(s).sum(axis=1) == np.abs(s[np.arange(H), s_h])).all()            # one non-zero score per head
    assert (np.abs(s[np.arange(H), s_h]) > 2).all()
    # sensitivity: the marked slot removed, moved to a neighbour, or rotated one position off
    alts = []
    s_rm = s.copy()
    s_rm[np.arange(H), s_h] = -np.inf
    alts.append(_softmax_out(lc, s_rm, q, native)[0])
    for dt in (-1, 1):
        t2 = np.clip(s_h + dt, 0, L - 1)
        s_mv = np.zeros_like(s)
        s_mv[np.arange(H), t2] = s[np.arange(H), s_h]
        moved = _softmax_out(lc, s_mv, q, native)[0]
        ok = t2 != s_h
        alts.append(np.where(ok[:, None], moved, np.inf))
    s_pos = np.zeros_like(s)
    for h in range(H):     # what the marked slot scores one position later
        if form == "dense":
            u = lut[h * 128:(h + 1) * 128, 1].double().numpy()
            s_pos[h, s_h[h]] = SCALE * (u * rq(h, s_h[h] + 1)).sum()
        else:
            c, val = mark[h]
            s_pos[h, s_h[h]] = SCALE * val * rq(h, s_h[h] + 1)[c]
    alts.append(_softmax_out(lc, s_pos, q, native)[0])
    tol = PROBE_TOL if precision == "fp32" else FP16_PROBE_TOL
    assert (_alt_err(want, alts) >= 10 * tol).all(), _alt_err(want, alts).min()
    o, l = _run(lc, q.astype(np.float32), precision=precision, native=native)
    _check("probe" if precision == "fp32" else "fp16_probe", o, want, tol,
           "%s bits=%d H=%d L=%d pos=%d %s" % (form, bits, H, L, pos_base, precision))
    if precision == "fp32":
        _check_lse(l, want_l)


@pytest.mark.parametrize("precision", ["fp32", "fp16"])
@pytest.mark.parametrize("form", ["dense", "outlier"])
@pytest.mark.parametrize("bits,H,L", [(4, 16, 4225), (4, 20, 1000), (3, 44, 2113), (3, 64, 481), (2, 8, 4225),
                                      (2, 36, 700)])
def test_marked_slot_probe(bits, H, L, form, precision):
    """Each head's marked slot at a boundary slot (K range, box, round, V tile, V CTA range, 0, L-1) at pos_offset 3."""
    L = min(L, _lmax())
    _marked_case(bits, H, L, form, 0, precision, n_sink=3)


@pytest.mark.parametrize("pos_end", [1234, 65536, 65537, (1 << 18) + 5])
@pytest.mark.parametrize("form", ["dense", "outlier"])
@pytest.mark.parametrize("bits,H", [(4, 24), (3, 52)])
def test_marked_slot_probe_at_large_positions(bits, H, form, pos_end):
    """L + pos_offset = 65536 gathers the outlier cos / sin from the table, 65537 evaluates them directly; a wrong
    position moves each head's marked score."""
    L = 500
    _marked_case(bits, H, L, form, pos_end - L, "fp32")
    _marked_case(bits, H, L, form, pos_end - L, "fp16")


@pytest.mark.parametrize("bits,H", [(4, 60), (3, 20), (2, 12)])
def test_marked_slot_probe_lut_form(bits, H):
    _marked_case(bits, H, 777, "dense", 0, "fp32", native=False)
    _marked_case(bits, H, 777, "outlier", 0, "fp32", native=False)


# ---- the legacy ops through the reference-compatible names -----------------------------------------------------------
@pytest.mark.parametrize("H", HS)
@pytest.mark.parametrize("bits", (4, 3, 2))
def test_legacy_v_op_every_head_count(bits, H):
    """vecquant{4,3,2}matmul_nuq_perchannel_transposed_mha_batched_fused_opt[2] at every (bits, H): with outlier rows
    (B = 1) and without (B = 2), against O.v_out_dense / v_out_outliers in float64."""
    from kvquant_b200 import quant_cuda as qc
    lc = _fill(_cache(bits, H), 300, seed=13)
    opt = getattr(qc, "vecquant%dmatmul_nuq_perchannel_transposed_mha_batched_fused_opt" % bits)
    opt2 = getattr(qc, "vecquant%dmatmul_nuq_perchannel_transposed_mha_batched_fused_opt2" % bits)
    vwords = lc.vcache.cpu().numpy().reshape(H * 4 * bits, -1)
    vlut = lc.vlut.cpu().numpy()
    for L in (300, 33):
        g = torch.Generator(device=DEV).manual_seed(L)
        p = torch.softmax(torch.randn((2, H, L), generator=g, device=DEV) * 2, -1).contiguous()
        pn = p.cpu().numpy()
        mul = torch.zeros((1, H, 128), device=DEV)
        opt2(p[:1].contiguous(), lc.vcache, mul, lc.vlut, L, lc.v_outliers, lc.v_outlier_idx)
        want = O.v_out_dense(pn[0], vwords, vlut, bits, L, H) + O.v_out_outliers(
            pn[0], lc.v_outliers.cpu().numpy(), lc.v_outlier_idx.cpu().numpy(), L, H)
        _check("legacy_v", mul[0].cpu().numpy(), want, EXACT_TOL, "opt2 bits=%d H=%d L=%d" % (bits, H, L))
        mul = torch.zeros((2, H, 128), device=DEV)
        opt(p, lc.vcache, mul, lc.vlut, L)
        for b in range(2):
            want = O.v_out_dense(pn[b], vwords, vlut, bits, L, H)
            _check("legacy_v", mul[b].cpu().numpy(), want, EXACT_TOL, "opt b=%d bits=%d H=%d L=%d" % (b, bits, H, L))


@pytest.mark.parametrize("H", HS)
@pytest.mark.parametrize("bits", (4, 3, 2))
def test_legacy_k_op_every_head_count(bits, H):
    """vecquant{4,3,2}matmul_nuq_perchannel_transposed_rope_mha_batched_fused_opt2 at every (bits, H): the 3-bit
    kernel's partial last head group at H != 0 mod 8, head counts that are not a multiple of a kernel's group."""
    from kvquant_b200 import quant_cuda as qc
    L, pos = 300, 3
    lc = _fill(_cache(bits, H), L, seed=14)
    q = _query(H, 4)
    mul = torch.zeros((1, H, L), device=DEV)
    getattr(qc, "vecquant%dmatmul_nuq_perchannel_transposed_rope_mha_batched_fused_opt2" % bits)(
        cu(q[None]), lc.kcache, mul, lc.klut.view(H, 128, -1), L, lc.k_outliers, lc.k_outlier_idx, THETA, pos)
    _check("legacy_k", mul[0].cpu().numpy(), _raw_scores(lc, L, q, pos), EXACT_TOL, "bits=%d H=%d" % (bits, H))
