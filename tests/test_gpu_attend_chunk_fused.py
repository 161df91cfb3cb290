"""kvq_attend_chunk / LayerCache.attend_chunk_fused: causal attention of a prompt chunk read straight from the
quantised cache (tensor-core kernel, K/V tiles dequantised in shared memory).

CPU: every argument error of the C entry point, T == 0 launches nothing, the scratch size is monotone.
GPU: against a float64 attention over exactly the kernel's fp16 operands (dequantize() of the slots, the sinks, the
chunk's fp16 rotated K/V, q rounded to fp16) at bits 4/3/2, 4..64 heads, sparse / dense-only / K-outliers-only
caches, Q-Norm, sinks and positions past 65536, across the T and L edges of the tiling and the key-split rule;
agreement with attend_chunk and with append-then-attend; causality and per-token sensitivity; determinism and
purity; a 1M-slot 7B-shaped cache within a memory bound that does not grow with the cache; a chunked prefill."""
import math

import numpy as np
import pytest
import torch

from _util import O, quantizer, rel_err, spec, synth

DEV = "cuda:0"
gpu = pytest.mark.gpu
NS, NO = 1.0625, -0.015625          # Q-Norm (normscale, normoffset)
BQ, BK = 128, 64                    # query rows per CTA, key tokens per tile (kvq_chunk.cu)
MAX_SPLITS, MAX_SMS = 32, 256

# float64 reference over the kernel's own operands: what is left is fp32 accumulation and the fp16 rounding of the
# softmax weights (2^-11 relative each).  Measured on an H100 SXM over the matrix of
# test_against_float64_over_the_kernel_operands, as the max over heads of max |got - ref| / max |ref| of that head:
# 6.0e-4 at most (a single query row, T = 1, where a few weights dominate), 1e-4 .. 3e-4 typically.  The tolerance
# is 3x the maximum.
MEASURED_MAX = 6.0e-4
TOL = 3 * MEASURED_MAX


def n_splits(T, H, L, sms):
    """The launcher's key-split rule (kvq_chunk.cu n_splits), restated: split the slot tiles over several CTAs per
    (query block, head) only when those CTAs fill at most half the SMs; at most one split per slot tile and 32 in
    all; the count is then trimmed so that every split owns at least one slot tile."""
    base = -(-T // BQ) * H
    tiles = -(-L // BK)
    sms = min(sms, MAX_SMS)
    if tiles < 2 or 2 * base > sms:
        return 1
    n = min(sms // base, tiles, MAX_SPLITS)
    per = -(-tiles // n)
    return -(-tiles // per)


def split_starts(T, H, L, sms):
    """First slot of each key split."""
    n = n_splits(T, H, L, sms)
    tiles = -(-L // BK)
    per = -(-tiles // n) if n > 1 else max(tiles, 1)
    return [s * per * BK for s in range(n)]


# ---------------------------------------------------------------------------------------------------------------------
# CPU
# ---------------------------------------------------------------------------------------------------------------------
def test_attend_chunk_argument_errors_without_a_gpu():
    from kvquant_b200 import _lib
    lib = _lib.load()
    P = 1 << 20                          # any 16-byte aligned non-NULL address: nothing is dereferenced on an error
    E_BITS, E_SHAPE, E_NULL, E_ALIGN = -1, -2, -3, -4
    good = dict(bits=4, H=32, Lmax=64, L=8, T=4, q=P, ck=P, cv=P, kcache=P, klut=P, k_out=P, k_idx=P, vcache=P,
                v_cent=P, v_aff=P, v_out=P, v_idx=P, n_out=42, rope=P, npos=64, pos_offset=0, sink_k=P, sink_v=P,
                n_sink=3, out=P, scratch=P)

    def call(**kw):
        a = dict(good, **kw)
        return lib.kvq_attend_chunk(a["bits"], a["H"], a["Lmax"], a["L"], a["T"], a["q"], a["ck"], a["cv"],
                                    a["kcache"], a["klut"], a["k_out"], a["k_idx"], a["vcache"], a["v_cent"],
                                    a["v_aff"], a["v_out"], a["v_idx"], a["n_out"], a["rope"], a["npos"],
                                    a["pos_offset"], a["sink_k"], a["sink_v"], a["n_sink"], a["out"], a["scratch"],
                                    None)
    assert call(bits=5) == E_BITS and call(bits=1) == E_BITS
    for kw in (dict(H=30), dict(H=0), dict(H=68), dict(Lmax=0, L=0), dict(L=-1), dict(L=65), dict(T=-1),
               dict(n_out=41), dict(n_out=130), dict(n_out=-2), dict(n_out=0), dict(npos=7), dict(pos_offset=57),
               dict(pos_offset=-1), dict(n_sink=-1)):
        assert call(**kw) == E_SHAPE, kw
    for kw in (dict(q=None), dict(ck=None), dict(cv=None), dict(out=None), dict(scratch=None), dict(kcache=None),
               dict(klut=None), dict(vcache=None), dict(v_cent=None), dict(v_aff=None), dict(rope=None),
               dict(k_out=None), dict(v_idx=None), dict(sink_k=None), dict(sink_v=None)):
        assert call(**kw) == E_NULL, kw
    for kw in (dict(q=P + 4), dict(ck=P + 8), dict(cv=P + 2), dict(out=P + 4), dict(scratch=P + 4)):
        assert call(**kw) == E_ALIGN, kw
    n0 = _lib.launch_count()
    assert call(T=0) == 0
    assert call(T=0, q=None, ck=None, cv=None, out=None, scratch=None) == 0    # nothing to attend: no pointer needed
    assert call(n_sink=0, sink_k=None, sink_v=None, T=0) == 0
    assert _lib.launch_count() == n0
    # valid without outliers (dense-only, K-only), without sinks, and with L == 0 (checked up to the first CUDA call)
    assert call(k_out=None, k_idx=None, v_out=None, v_idx=None, T=0) == 0
    assert call(v_out=None, v_idx=None, n_sink=0, sink_k=None, sink_v=None, L=0, T=0) == 0


def test_scratch_size_is_monotone_and_device_independent():
    from kvquant_b200 import _lib
    lib = _lib.load()
    f = lib.kvq_attend_chunk_scratch_bytes
    assert f(32, 0, 1000) == 0
    for H in (4, 32, 40, 64):
        Ts = [1, 2, 15, 16, 17, 127, 128, 129, 300, 2048, 65536]
        Ls = [0, 1, 63, 64, 65, 1000, 2048, 131072, 1 << 20]
        grid = np.array([[f(H, T, L) for L in Ls] for T in Ts], dtype=np.int64)
        assert np.all(np.diff(grid, axis=0) >= 0) and np.all(np.diff(grid, axis=1) >= 0), H
        # large enough for the partials of every split count the launcher can pick on any device
        for T in Ts:
            for L in Ls:
                n = max(n_splits(T, H, L, sms) for sms in (16, 78, 114, 132, 144, 170, 256, 1024))
                if n > 1:
                    assert f(H, T, L) >= n * T * H * 130 * 4, (H, T, L)


def test_split_rule_restatement_changes_with_length():
    """The split counts the GPU tests rely on (132 SMs): several values along L at small T, one at large T."""
    assert [n_splits(1, 32, L, 132) for L in (0, 64, 65, 129, 193, 1000)] == [1, 1, 2, 3, 4, 4]
    assert n_splits(1, 4, 1000, 132) == 16 and n_splits(1, 4, 1 << 20, 132) == 32
    assert n_splits(512, 32, 1 << 20, 132) == 1 and n_splits(2048, 4, 1000, 132) == 2
    assert n_splits(300, 4, 1000, 132) == 8 and n_splits(130, 4, 1000, 132) == 16


# ---------------------------------------------------------------------------------------------------------------------
# GPU helpers
# ---------------------------------------------------------------------------------------------------------------------
def cu(x):
    return torch.from_numpy(np.ascontiguousarray(x)).to(DEV)


_CACHES = {}


def filled_cache(bits, H, mode="kv", qnorm=False, L=1000, Lmax=None):
    """LayerCache with L synthetic tokens appended in chunks (append_chunk).  mode: "kv" (K and V outliers),
    "dense" (dense-only), "k_only" (K outliers only)."""
    key = (bits, H, mode, qnorm, L)
    if key in _CACHES:
        lc = _CACHES[key]
        lc.len, lc.n_sink, lc.pos_base, lc.sink_k, lc.sink_v = L, 0, 0, None, None
        return lc
    from kvquant_b200.cache import LayerCache
    klut, vcent = quantizer(bits, H)
    if qnorm:
        cal = synth.calibrate(spec(H), bits, calib_tokens=512, seed=7)
        klut = O.build_k_lut(cal["k"][0], cal["k"][1], cal["k"][2][0], normscale=NS, normoffset=NO)
    lc = LayerCache.from_luts(bits, H, Lmax or (L + 64), klut, vcent, device=DEV, include_sparse=mode != "dense",
                              sparse_v=mode == "kv", v_norm=(NS, NO) if qnorm else None)
    k, v = cu(spec(H).k_tokens(L, seed=21)), cu(spec(H).v_tokens(L, seed=22))
    for s0 in range(0, L, 512):
        lc.append_chunk(k[s0:s0 + 512], v[s0:s0 + 512])
    assert lc.len == L
    _CACHES[key] = lc
    return lc


def set_sinks(lc, n_sink, seed=4):
    lc.n_sink = n_sink
    if n_sink:
        g = torch.Generator(device=DEV).manual_seed(seed)
        lc.set_sinks(torch.randn((lc.H, 128, n_sink), generator=g, device=DEV).half(),
                     torch.randn((lc.H, n_sink, 128), generator=g, device=DEV).half())
    else:
        lc.sink_k = lc.sink_v = None


def chunk_inputs(H, T, seed):
    """q f32 [T, H, 128] (fp16-representable, as from an fp16 projection), k / v f32 [T, hidden]."""
    sp = spec(H)
    rng = np.random.default_rng([seed, 9])
    q = rng.standard_normal((T, H, 128)).astype(np.float16).astype(np.float32)
    return cu(q), cu(sp.k_tokens(T, seed=31 + seed)), cu(sp.v_tokens(T, seed=32 + seed))


def operands(lc, k, v, theta, L=None):
    """The kernel's fp16 operands: [sinks | dequantize(0, L, theta) | chunk rotated K / V], each [H, S, 128]."""
    L = lc.len if L is None else L
    T = k.shape[0]
    ns = lc.n_sink if lc.sink_k is not None else 0
    kc = torch.empty((lc.H, T, 128), dtype=torch.float16, device=DEV)
    vc = torch.empty_like(kc)
    lc._chunk_kv16(k, v, theta, lc.n_sink + lc.pos_base + L, kc, vc)
    ks, vs = lc.dequantize(0, L, theta)
    parts_k, parts_v = [ks, kc], [vs, vc]
    if ns:
        parts_k.insert(0, lc.sink_k.transpose(1, 2))
        parts_v.insert(0, lc.sink_v)
    return torch.cat(parts_k, 1), torch.cat(parts_v, 1), ns


def reference(lc, q, k, v, theta, rows=None):
    """float64 causal softmax(q16 K^T / sqrt(128)) V over the kernel's operands, head by head.  [T or rows, H, 128]."""
    K, V, ns = operands(lc, k, v, theta)
    L, T = lc.len, q.shape[0]
    rows = torch.arange(T, device=DEV) if rows is None else torch.as_tensor(rows, device=DEV)
    q16 = q[rows].half().double()
    allowed = torch.arange(K.shape[1], device=DEV)[None, :] <= (ns + L + rows)[:, None]
    out = torch.empty((len(rows), lc.H, 128), dtype=torch.float64, device=DEV)
    for h in range(lc.H):
        s = q16[:, h] @ K[h].double().t() / math.sqrt(128)
        s = s.masked_fill(~allowed, float("-inf"))
        out[:, h] = torch.softmax(s, -1) @ V[h].double()
    return out


def head_err(got, want):
    """max over heads of max |got - want| / max |want| (per head)."""
    d = (got.double() - want).abs().amax(dim=(0, 2))
    return float((d / want.abs().amax(dim=(0, 2)).clamp_min(1e-30)).max())


# ---------------------------------------------------------------------------------------------------------------------
# GPU: float64 reference
# ---------------------------------------------------------------------------------------------------------------------
# (bits, H, mode, qnorm, n_sink, pos_base)
CONFIGS = [(4, 32, "kv", False, 0, 0), (3, 32, "kv", False, 5, 0), (2, 32, "kv", False, 0, 70_000),
           (4, 4, "kv", False, 5, 0), (4, 40, "dense", False, 0, 0), (4, 64, "k_only", False, 5, 65_530),
           (2, 32, "kv", True, 5, 0), (4, 32, "kv", True, 0, 0), (3, 40, "k_only", False, 0, 0),
           (2, 64, "dense", False, 5, 0), (4, 4, "kv", False, 130, 0), (3, 32, "k_only", False, 64, 70_000)]
# (T, L): every T edge of the query blocks and every L edge of the key tiles, and lengths where the split count
# changes (at T = 1, 32 heads: 1, 1, 2, 3, 4 splits for L = 0, 64, 65, 129, 193)
SHAPES = [(1, 1000), (15, 0), (16, 1), (17, 63), (BQ - 1, 64), (BQ, 65), (BQ + 1, 1000), (300, 1000), (2048, 1000),
          (1, 64), (1, 65), (1, 129), (1, 193), (64, 1000)]


@gpu
@pytest.mark.parametrize("bits,H,mode,qnorm,n_sink,pos_base", CONFIGS)
def test_against_float64_over_the_kernel_operands(bits, H, mode, qnorm, n_sink, pos_base):
    theta = 10000.0 if bits != 3 else 1e6
    lc = filled_cache(bits, H, mode, qnorm)
    set_sinks(lc, n_sink)
    lc.pos_base = pos_base
    sms = torch.cuda.get_device_properties(DEV).multi_processor_count
    seen = set()
    for i, (T, L) in enumerate(SHAPES):
        lc.len = L
        q, k, v = chunk_inputs(H, T, seed=i)
        got = lc.attend_chunk_fused(q, k, v, rope_theta=theta)
        assert got.shape == (T, H, 128) and got.dtype == torch.float32
        err = head_err(got, reference(lc, q, k, v, theta))
        assert err < TOL, (T, L, err)
        seen.add(n_splits(T, H, L, sms))
    assert len(seen) >= 2, seen          # one and several key splits were exercised
    lc.len = 1000


# ---------------------------------------------------------------------------------------------------------------------
# GPU: agreement with the existing paths
# ---------------------------------------------------------------------------------------------------------------------
@gpu
@pytest.mark.parametrize("bits,H,mode,n_sink", [(4, 32, "kv", 0), (3, 32, "kv", 4), (2, 40, "k_only", 4)])
@pytest.mark.parametrize("T", [1, 64, 300])
def test_agrees_with_attend_chunk(bits, H, mode, n_sink, T):
    lc = filled_cache(bits, H, mode)
    set_sinks(lc, n_sink)
    q, k, v = chunk_inputs(H, T, seed=40 + T)
    got = lc.attend_chunk_fused(q, k, v)
    want = lc.attend_chunk(q, k, v)
    assert rel_err(got.cpu().numpy(), want.cpu().numpy())[0] < 4e-3


@gpu
def test_one_token_equals_append_then_attend():
    """T = 1 is one decode step (the tolerance of attend_chunk's own test: the appended token is quantised there)."""
    bits, H, L, theta = 4, 32, 1000, 10000.0
    lc = filled_cache(bits, H)
    sp = spec(H)
    q = cu(O.rope_rotate_q(sp.q_vec(77), L, theta))
    k, v = cu(sp.k_tokens(1, seed=78)), cu(sp.v_tokens(1, seed=79))
    got = lc.attend_chunk_fused(q[None], k, v, rope_theta=theta)[0]
    from kvquant_b200.cache import LayerCache
    lc2 = LayerCache.from_luts(bits, H, lc.Lmax, *quantizer(bits, H), device=DEV)
    kk, vv = cu(sp.k_tokens(L, seed=21)), cu(sp.v_tokens(L, seed=22))
    for s0 in range(0, L, 512):
        lc2.append_chunk(kk[s0:s0 + 512], vv[s0:s0 + 512])
    lc2.append(k[0], v[0])
    lc2.precision = "fp32"
    want = lc2.attend(q)
    assert rel_err(got.cpu().numpy(), want.cpu().numpy())[0] < 1e-2


# ---------------------------------------------------------------------------------------------------------------------
# GPU: causality and coverage, determinism and purity
# ---------------------------------------------------------------------------------------------------------------------
@gpu
@pytest.mark.parametrize("H,T", [(4, 300), (32, 300)])      # 4 heads: 8 key splits; 32 heads: one
def test_later_chunk_tokens_do_not_reach_earlier_rows(H, T):
    lc = filled_cache(4, H)
    set_sinks(lc, 5)
    q, k, v = chunk_inputs(H, T, seed=5)
    a = lc.attend_chunk_fused(q, k, v)
    for i in (0, 63, 64, 127, 128, 200):
        q2, k2, v2 = q.clone(), k.clone(), v.clone()
        q2[i + 1:] += 1.0
        k2[i + 1:] *= -2.0
        v2[i + 1:] += 3.0
        b = lc.attend_chunk_fused(q2, k2, v2)
        assert torch.equal(a[:i + 1], b[:i + 1]), i
        assert not torch.equal(a[i + 1:], b[i + 1:]), i


@gpu
def test_each_region_reaches_the_output_as_float64_predicts():
    """Adding 1000 to one token's V moves the output by what the float64 reference predicts, for the first and last
    sink, slot 0, slot L-1, the first slot of every key split, chunk token 0 and the diagonal token."""
    H, T, L, ns, theta = 4, 130, 1000, 5, 10000.0
    lc = filled_cache(4, H)
    set_sinks(lc, ns)
    sms = torch.cuda.get_device_properties(DEV).multi_processor_count
    starts = split_starts(T, H, L, sms)
    assert len(starts) > 1
    q, k, v = chunk_inputs(H, T, seed=6)
    base_got = lc.attend_chunk_fused(q, k, v)
    base_ref = reference(lc, q, k, v, theta)
    scale = base_ref.abs().max().item()
    probes = [("sink", 0), ("sink", ns - 1), ("slot", 0), ("slot", L - 1)] + [("slot", s) for s in starts[1:]] + \
             [("chunk", 0), ("chunk", 77)]
    vaff0, sink_v0 = lc.vaff.clone(), lc.sink_v.clone()
    try:
        for kind, j in probes:
            v2 = v
            if kind == "sink":
                lc.sink_v[:, j] += 1000.0
            elif kind == "slot":
                lc.vaff[j, 1] += 1000.0
            else:
                v2 = v.clone()
                v2[j] += 1000.0
            dg = lc.attend_chunk_fused(q, k, v2).double() - base_got.double()
            dr = reference(lc, q, k, v2, theta) - base_ref
            felt = dr.abs().max().item()
            assert felt > 20 * TOL * scale, (kind, j, felt, scale)       # the probe is felt
            # both outputs carry their own error, relative to the larger outputs after the change
            assert (dg - dr).abs().max().item() < 2 * TOL * (scale + felt), (kind, j, (dg - dr).abs().max().item())
            if kind == "chunk":
                assert torch.equal(dg[:j], torch.zeros_like(dg[:j]))     # rows before the token never see it
            lc.vaff.copy_(vaff0)
            lc.sink_v.copy_(sink_v0)
    finally:
        lc.vaff.copy_(vaff0)
        lc.sink_v.copy_(sink_v0)


@gpu
@pytest.mark.parametrize("H,T", [(4, 1), (4, 300), (32, 300), (64, 17)])
def test_deterministic_and_pure(H, T):
    lc = filled_cache(3, H)
    set_sinks(lc, 3)
    names = ("kcache", "vcache", "vaff", "vlut", "k_outliers", "k_outlier_idx", "v_outliers", "v_outlier_idx",
             "sink_k", "sink_v")
    before = {n: getattr(lc, n).clone() for n in names}
    q, k, v = chunk_inputs(H, T, seed=7)
    a = lc.attend_chunk_fused(q, k, v)
    b = lc.attend_chunk_fused(q, k, v)
    assert torch.equal(a.view(torch.int32), b.view(torch.int32))
    for n in names:
        assert torch.equal(getattr(lc, n), before[n]), n
    assert lc.len == 1000


@gpu
def test_refuses_what_attend_chunk_refuses():
    lc = filled_cache(4, 4)
    q, k, v = chunk_inputs(4, 8, seed=8)
    with pytest.raises(ValueError):
        lc.attend_chunk_fused(q[:, :2], k, v)
    with pytest.raises(ValueError):
        lc.attend_chunk_fused(q, k[:4], v)
    with pytest.raises(TypeError):
        lc.attend_chunk_fused(q.double(), k, v)
    lc.use_native_v = False
    try:
        with pytest.raises(NotImplementedError):
            lc.attend_chunk_fused(q, k, v)
    finally:
        lc.use_native_v = True


# ---------------------------------------------------------------------------------------------------------------------
# GPU: a 1M-slot cache, the capability itself
# ---------------------------------------------------------------------------------------------------------------------
@gpu
def test_million_slot_cache_within_a_memory_bound_that_does_not_grow_with_it():
    from kvquant_b200.cache import LayerCache
    bits, H, L, T, theta = 4, 32, 1 << 20, 512, 10000.0
    klut, vcent = quantizer(bits, H)
    lc = LayerCache.from_luts(bits, H, L, klut, vcent, device=DEV, include_sparse=False)
    g = torch.Generator(device=DEV).manual_seed(5)
    for t in (lc.kcache, lc.vcache):
        t.copy_(torch.randint(-2 ** 31, 2 ** 31, t.shape, generator=g, device=DEV, dtype=torch.int64).to(torch.int32))
    lc.vaff[:, 0] = torch.rand(L, generator=g, device=DEV) + 0.5
    lc.vaff[:, 1] = torch.rand(L, generator=g, device=DEV) - 0.5
    lc.len = L
    q, k, v = chunk_inputs(H, T, seed=11)
    from kvquant_b200 import quant_cuda as qc
    qc.rope_tables(lc.device, theta, L + T)                                   # the 1M-position rope table, built once
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats(DEV)
    m0 = torch.cuda.memory_allocated(DEV)
    got = lc.attend_chunk_fused(q, k, v, rope_theta=theta)
    torch.cuda.synchronize()
    grew = torch.cuda.max_memory_allocated(DEV) - m0
    kv16 = 2 * H * T * 128 * 2
    scratch = lc.lib.kvq_attend_chunk_scratch_bytes(H, T, L)
    # the chunk's fp16 K/V, the scratch, the f32 output and the f32 rotation temporaries of the chunk's keys
    bound = kv16 + scratch + T * H * 128 * 4 + 4 * T * H * 128 * 4
    materialised = 2 * H * (L + T) * 128 * 2
    assert grew <= bound, (grew, bound)
    assert bound < materialised / 200, (bound, materialised)     # attend_chunk would need 16 GiB more

    # float64 reference for a sample of rows, all heads, streamed over slot ranges (no full-cache buffer)
    rows = torch.tensor([0, 1, 255, 256, 511], device=DEV)
    q16 = q[rows].half().double()                                            # [R, H, 128]
    m = torch.full((len(rows), H), float("-inf"), dtype=torch.float64, device=DEV)
    den = torch.zeros((len(rows), H), dtype=torch.float64, device=DEV)
    num = torch.zeros((len(rows), H, 128), dtype=torch.float64, device=DEV)

    def fold(Kp, Vp, mask=None):                                             # Kp, Vp [H, n, 128]
        nonlocal m, den, num
        s = torch.einsum("rhc,hnc->rhn", q16, Kp.double()) / math.sqrt(128)
        if mask is not None:
            s = s.masked_fill(~mask[:, None, :], float("-inf"))
        m2 = torch.maximum(m, s.amax(-1))
        c = torch.exp(m - m2)
        p = torch.exp(s - m2[..., None])
        den = den * c + p.sum(-1)
        num = num * c[..., None] + torch.einsum("rhn,hnc->rhc", p, Vp.double())
        m = m2
    step = 1 << 16
    for s0 in range(0, L, step):
        fold(*lc.dequantize(s0, s0 + step, theta))
    kc = torch.empty((H, T, 128), dtype=torch.float16, device=DEV)
    vc = torch.empty_like(kc)
    lc._chunk_kv16(k, v, theta, L, kc, vc)
    fold(kc, vc, torch.arange(T, device=DEV)[None, :] <= rows[:, None])
    want = num / den[..., None]
    err = head_err(got[rows], want)
    # random codes and (sf, off) centred on 0: each row averages ~1M near-uniformly weighted values of either sign, so
    # max |out| is small against the values summed and the relative error larger (measured 1.5e-3 on an H100 SXM)
    assert err < 3e-3, err


# ---------------------------------------------------------------------------------------------------------------------
# GPU: prefill-shaped use
# ---------------------------------------------------------------------------------------------------------------------
@gpu
@pytest.mark.parametrize("n_sink", [0, 3])
def test_chunked_prefill_on_the_fused_attend_matches_prefill(n_sink):
    """One layer: its cache depends on the prompt alone, so the two loops differ only in the attention numerics.  (A
    second layer quantises K/V computed from the first layer's attention output, where a last-bit difference can flip a
    4-bit code; two layers at n_sink = 3 were measured 1.2e-2 apart, against 1e-2 here.)"""
    from kvquant_b200 import decode as kd, cache as kc
    from kvquant_b200.decode import rmsnorm
    cfg = kd.DecodeConfig(n_layers=1, hidden=4096, n_heads=32, intermediate=1024, vocab=512, bits=4, n_sink=n_sink,
                          max_len=512)
    cal = synth.calibrate(spec(32), 4, calib_tokens=256, seed=7)
    t = kc.build_k_lookup_table(cal["k"][0], cal["k"][1], cal["k"][2][0], 32, device=DEV)
    quant = dict(klut=dict(lut=t["lut"], lut2=None, thr_lower=t["thr_lower"], thr_upper=t["thr_upper"]),
                 v_cent=cal["v"][2][0])
    st = kd.DecoderStage(cfg, 0, 1, DEV, quant, seed=1, with_head=True)
    g = torch.Generator(device=DEV).manual_seed(2)
    x = (torch.randn((300, cfg.hidden), generator=g, device=DEV) * 0.5).half()
    want = st.prefill(x, chunk=128)
    for ly in st.layers:
        ly.cache.reset()
    H, hid = cfg.n_heads, cfg.hidden
    outs = []
    for s0 in range(0, x.shape[0], 128):
        h = x[s0:s0 + 128]
        n = h.shape[0]
        for ly in st.layers:
            c = ly.cache
            q, k, v = (rmsnorm(h, ly.n1, cfg.rms_eps) @ ly.wqkv.t()).float().split(hid, dim=-1)
            q = st._rope_rows(q.reshape(n, H, 128), c.n_sink + c.len + torch.arange(n, device=DEV)).contiguous()
            k, v = k.contiguous(), v.contiguous()
            o = c.attend_chunk_fused(q, k, v, rope_theta=cfg.rope_theta)
            c.append_chunk(k, v)
            h = h + o.half().view(n, hid) @ ly.wo.t()
            gg, u = (rmsnorm(h, ly.n2, cfg.rms_eps) @ ly.wgu.t()).split(cfg.intermediate, dim=-1)
            h = h + (torch.nn.functional.silu(gg) * u) @ ly.wdown.t()
        outs.append(h)
    got = torch.cat(outs)
    assert all(ly.cache.len == 300 for ly in st.layers)
    d = (got.float() - want.float()).abs().max().item()
    assert d <= 1e-2 * max(1.0, want.float().abs().max().item()), d
