"""kvq_dequant_kv / LayerCache.dequantize / LayerCache.attend_chunk: the quantised cache read back on the device.

CPU: every argument error of the C entry point (returned before any CUDA call), and the rotate-half convention of the
rotated K output pinned against the oracle's K scores.
GPU: pre-RoPE K bit-exact and V within one fp16 ulp (plus the oracle table's own rounding) of the oracle's reconstruction (bits 4/3/2, 40 and 64 heads,
sparse / dense-only / K-outliers-only caches, K and V Q-Norm, several slot ranges); rotated K against a float64
rotation; the fused attend reproduced from the dequantised cache; in-place writes into a larger buffer; 64-bit output
offsets past 2^31 elements; the chunked causal attention against a float64 reference."""
import ctypes
import math

import numpy as np
import pytest
import torch

from _util import O, oracle_cache, quantizer, rel_err, spec, synth

DEV = "cuda:0"
gpu = pytest.mark.gpu
NS, NO = 1.0625, -0.015625          # Q-Norm (normscale, normoffset)


# ---------------------------------------------------------------------------------------------------------------------
# reference reconstruction (float64 unless stated), with the tables the decode path dequantises with
# ---------------------------------------------------------------------------------------------------------------------
def k_recon(c, dtype=np.float64):
    """K of an OracleCache [hidden, L]: dequantisation table (LUT2 under Q-Norm, as k_scores uses) plus the outlier
    residual, added in `dtype` (float32: one fp32 add, as the device computes it)."""
    deq = c.klut["lut2"] if c.klut.get("lut2") is not None else c.klut["lut"]
    kk = O.k_dequant(c.kwords[:, :c.len], deq, c.bits).astype(dtype)
    if c.sparse:
        idx, val = c.k_idx[:c.len].astype(np.int64), c.k_out[:c.len]
        t = np.broadcast_to(np.arange(c.len)[:, None], idx.shape)
        nz = val != 0
        np.add.at(kk, (idx[nz], t[nz]), val[nz].astype(dtype))     # at most one non-zero residual per (channel, slot)
    return kk


def v_recon(c):
    """V of an OracleCache: the per-token table (the Q-Norm one when V Q-Norm is on) plus the outlier residual.
    float64 [hidden, L]."""
    lut = c.vlut2 if c.v_norm is not None else c.vlut
    vv = O.v_dequant(c.vwords[:, :c.len], lut[:c.len], c.bits).astype(np.float64)
    if c.sparse_v:
        t = np.broadcast_to(np.arange(c.len)[:, None], c.v_idx[:c.len].shape)
        np.add.at(vv, (c.v_idx[:c.len].astype(np.int64), t), c.v_out[:c.len].astype(np.float64))
    return vv


def rotate_k(kk, positions, rope_theta):
    """Rotate-half RoPE of K [hidden, n] (float64) at `positions` [n], with the cos/sin the decode kernels use:
    k'[c] = cos*k[c] - sin*k[c+64] (c < 64), cos*k[c] + sin*k[c-64] (c >= 64)."""
    hidden, n = kk.shape
    k = np.asarray(kk, dtype=np.float64).reshape(hidden // 128, 128, n)
    cos, sin = O.rope_cos_sin(O.rope_theta_vec(rope_theta), positions)     # [n, 128], channel c and c ^ 64 equal
    cos, sin = cos.T[None], sin.T[None]
    partner = np.concatenate([-k[:, 64:], k[:, :64]], axis=1)
    return (k * cos + partner * sin).reshape(hidden, n)


def head_major(x, H):
    """[hidden, n] -> [H, n, 128]."""
    return np.ascontiguousarray(np.asarray(x).reshape(H, 128, -1).transpose(0, 2, 1))


# ---------------------------------------------------------------------------------------------------------------------
# CPU
# ---------------------------------------------------------------------------------------------------------------------
def test_dequant_argument_errors_without_a_gpu():
    from kvquant_b200 import _lib
    lib = _lib.load()
    P = 1 << 20                          # any 16-byte aligned non-NULL address: nothing is dereferenced on an error
    E_BITS, E_SHAPE, E_NULL, E_ALIGN = -1, -2, -3, -4
    good = dict(bits=4, H=32, Lmax=64, start=0, stop=8, kcache=P, klut=P, k_out=P, k_idx=P, vcache=P, v_cent=P,
                v_aff=P, v_out=P, v_idx=P, n_out=42, rope=P, npos=64, pos_offset=0, out_k=P, out_v=P,
                head_stride=8 * 128)

    def call(**kw):
        a = dict(good, **kw)
        return lib.kvq_dequant_kv(a["bits"], a["H"], a["Lmax"], a["start"], a["stop"], a["kcache"], a["klut"],
                                  a["k_out"], a["k_idx"], a["vcache"], a["v_cent"], a["v_aff"], a["v_out"], a["v_idx"],
                                  a["n_out"], a["rope"], a["npos"], a["pos_offset"], a["out_k"], a["out_v"],
                                  a["head_stride"], None)
    assert call(bits=5) == E_BITS and call(bits=1) == E_BITS
    for kw in (dict(start=9), dict(start=-1, stop=0), dict(stop=65), dict(H=30), dict(H=0), dict(H=68), dict(n_out=41),
               dict(n_out=130), dict(n_out=0), dict(head_stride=8 * 128 - 8), dict(npos=7),
               dict(pos_offset=57), dict(pos_offset=-1), dict(Lmax=0, stop=0)):
        assert call(**kw) == E_SHAPE, kw
    for kw in (dict(kcache=None), dict(klut=None), dict(vcache=None), dict(v_cent=None), dict(v_aff=None),
               dict(out_k=None, out_v=None), dict(k_out=None), dict(v_idx=None)):
        assert call(**kw) == E_NULL, kw
    for kw in (dict(out_k=P + 8), dict(out_v=P + 2), dict(head_stride=8 * 128 + 4)):
        assert call(**kw) == E_ALIGN, kw
    # a side that is not requested needs none of its pointers; the rope table is checked only for K
    n0 = _lib.launch_count()
    assert call(start=3, stop=3, out_k=None, kcache=None, klut=None, rope=None) == 0      # empty range: no launch
    assert call(start=8, stop=8, out_v=None, vcache=None, v_cent=None, v_aff=None) == 0
    assert call(start=0, stop=0, head_stride=0) == 0
    assert call(start=4, stop=4, out_k=None, out_v=None, kcache=None, vcache=None) == 0   # zero-element outputs: NULL
    assert call(start=4, stop=4, out_k=P + 2) == 0
    assert _lib.launch_count() == n0
    assert lib.kvq_error_string(E_SHAPE)


@pytest.mark.parametrize("qnorm", [False, True])
def test_rotated_recon_reproduces_the_oracle_k_scores(qnorm):
    """q_rot . rotate(k_recon)[:, t] == k_scores(q)[:, t] to float64 rounding: the convention of the rotated output
    (and, under Q-Norm, that K is reconstructed with the table the scores use)."""
    bits, H, L, pos_offset, theta = 2 if qnorm else 4, 32, 40, 7, 10000.0
    klut, vcent = quantizer(bits, H)
    if qnorm:
        cal = synth.calibrate(spec(H), bits, calib_tokens=512, seed=7)
        klut = O.build_k_lut(cal["k"][0], cal["k"][1], cal["k"][2][0], normscale=NS, normoffset=NO)
    c = O.OracleCache(bits, H, 64, klut, vcent, v_norm=(NS, NO) if qnorm else None)
    k, v = spec(H).k_tokens(L, seed=3), spec(H).v_tokens(L, seed=4)
    for t in range(L):
        c.append(k[t], v[t])
    q = O.rope_rotate_q(spec(H).q_vec(5), L + pos_offset, theta).astype(np.float64)
    want = c.k_scores(q, theta, pos_offset)
    kr = rotate_k(k_recon(c), np.arange(L) + pos_offset, theta).reshape(H, 128, L)
    got = np.einsum("hc,hct->ht", q, kr)
    scale = np.abs(q)[:, :, None] * np.abs(kr)
    assert np.all(np.abs(got - want) <= 1e-13 * scale.sum(axis=1)), np.abs(got - want).max()


# ---------------------------------------------------------------------------------------------------------------------
# GPU
# ---------------------------------------------------------------------------------------------------------------------
def cu(x):
    return torch.from_numpy(np.ascontiguousarray(x)).to(DEV)


_CACHES = {}


def appended_cache(bits, H, L, mode="kv", qnorm=False):
    """(OracleCache, LayerCache) with the same L tokens, the device one filled through the fused append.
    mode: "kv" (K and V outliers), "dense" (dense-only), "k_only" (K outliers only)."""
    key = (bits, H, L, mode, qnorm)
    if key in _CACHES:
        return _CACHES[key]
    from kvquant_b200.cache import LayerCache
    klut, vcent = quantizer(bits, H)
    if qnorm:
        cal = synth.calibrate(spec(H), bits, calib_tokens=512, seed=7)
        klut = O.build_k_lut(cal["k"][0], cal["k"][1], cal["k"][2][0], normscale=NS, normoffset=NO)
    sparse, sparse_v = mode != "dense", mode == "kv"
    vn = (NS, NO) if qnorm else None
    Lmax = (L + 63) // 64 * 64 + 64
    c = O.OracleCache(bits, H, Lmax, klut, vcent, include_sparse=sparse, sparse_v=sparse_v, v_norm=vn)
    lc = LayerCache.from_luts(bits, H, Lmax, klut, vcent, device=DEV, include_sparse=sparse, sparse_v=sparse_v,
                              v_norm=vn)
    k, v = spec(H).k_tokens(L, seed=21), spec(H).v_tokens(L, seed=22)
    kd, vd = cu(k), cu(v)
    for t in range(L):
        c.append(k[t], v[t])
        lc.append(kd[t], vd[t])
    assert np.array_equal(lc.kcache.cpu().numpy().reshape(-1, Lmax), c.kwords)
    assert np.array_equal(lc.vcache.cpu().numpy().reshape(-1, Lmax), c.vwords)
    _CACHES[key] = (c, lc)
    return c, lc


def fp16_ulp(x):
    return np.spacing(np.abs(np.asarray(x, dtype=np.float16))).astype(np.float64)


def v_table_err(c):
    """Rounding of the oracle's per-token table entry cent*sf + off (two fp32 roundings, where the kernel's fma has
    one): 2 fp32 ulps of |cent*sf| + |off|, [hidden, L].  Next to zero it exceeds an fp16 ulp of the result when a
    token's range is wide (dense-only V keeps the heavy-tail values: sf ~ 100)."""
    cent = c.v_cent2 if c.v_norm is not None else c.v_cent
    codes = O.unpack_codes(c.vwords[:, :c.len], c.bits).astype(np.int64)
    sf, off = c.vaff[:c.len, 0].astype(np.float64), c.vaff[:c.len, 1].astype(np.float64)
    mag = np.abs(cent.astype(np.float64)[codes] * sf) + np.abs(off)
    return 2 * np.spacing(mag.astype(np.float32)).astype(np.float64)


CONFIGS = [(4, 32, "kv", False), (3, 32, "kv", False), (2, 32, "kv", False), (4, 40, "kv", False),
           (4, 64, "kv", False), (4, 32, "dense", False), (4, 32, "k_only", False), (2, 32, "kv", True),
           (4, 32, "kv", True)]


@gpu
@pytest.mark.parametrize("bits,H,mode,qnorm", CONFIGS)
def test_prerope_k_bit_exact_and_v_within_one_ulp(bits, H, mode, qnorm):
    L = 1000
    c, lc = appended_cache(bits, H, L, mode, qnorm)
    kw = head_major(k_recon(c, np.float32), H).astype(np.float16)
    vw = head_major(v_recon(c), H)
    vtol = head_major(v_table_err(c), H)
    for start, stop in ((0, 1), (5, 37), (31, L), (L - 1, L), (45, 300), (0, L)):
        k, v = lc.dequantize(start, stop)
        assert k.shape == v.shape == (H, stop - start, 128) and k.dtype == v.dtype == torch.float16
        k, v = k.cpu().numpy(), v.cpu().numpy()
        assert np.array_equal(k, kw[:, start:stop]), (start, stop, np.argwhere(k != kw[:, start:stop])[:5])
        want = vw[:, start:stop]
        d = np.abs(v.astype(np.float64) - want.astype(np.float16).astype(np.float64))
        assert np.all(d <= fp16_ulp(want) + vtol[:, start:stop]), (start, stop, d.max())
    k, _ = lc.dequantize()                                   # stop defaults to len
    assert k.shape[1] == L
    if mode != "dense":
        assert np.count_nonzero(c.k_out[:L]) > L            # the residuals were exercised


@gpu
@pytest.mark.parametrize("bits,H,n_sink,pos_base,theta", [(4, 32, 5, 0, 10000.0), (4, 32, 0, 1234, 10000.0),
                                                          (3, 40, 5, 77, 1e6), (2, 32, 0, 0, 1e6)])
def test_rotated_k_against_float64_rotation(bits, H, n_sink, pos_base, theta):
    L = 1000
    c, lc = appended_cache(bits, H, L)
    lc.n_sink, lc.pos_base = n_sink, pos_base
    try:
        kk = k_recon(c)
        for start, stop in ((0, L), (37, 70), (L - 1, L)):
            got = lc.dequantize(start, stop, rope_theta=theta)[0].cpu().numpy().astype(np.float64)
            pos = np.arange(start, stop) + n_sink + pos_base
            want = head_major(rotate_k(kk[:, start:stop], pos, theta), H)
            mag = head_major(kk[:, start:stop], H)
            mag = np.maximum(np.abs(mag), np.abs(np.concatenate([mag[..., 64:], mag[..., :64]], axis=-1)))
            d = np.abs(got - want)
            # the device table's frequencies come from CUDA powf, which may differ from the float64 pow by one fp32 ulp
            # (theta_j <= 1): an angle error of up to 2.4e-7 * p radians on a pair of magnitude `mag`
            tol = fp16_ulp(np.maximum(mag, np.abs(want))) + 2.4e-7 * pos[None, :, None] * mag
            assert np.all(d <= tol), (start, stop, d.max())
    finally:
        lc.n_sink, lc.pos_base = 0, 0


@gpu
@pytest.mark.parametrize("bits,H,mode", [(4, 32, "kv"), (3, 32, "kv"), (4, 40, "k_only"), (2, 32, "dense")])
@pytest.mark.parametrize("n_sink", [0, 5])
def test_sdpa_over_the_dequantised_cache_matches_the_fused_attend(bits, H, mode, n_sink):
    """fp32 SDPA (math backend) of one rotated query over [sinks | dequantize(rope_theta)] == LayerCache.attend.  The
    difference is the fp16 rounding of the dequantised K and V (2^-11 relative per element)."""
    from torch.nn.attention import SDPBackend, sdpa_kernel
    L, theta = 1000, 10000.0
    c, lc = appended_cache(bits, H, L, mode)
    sp = spec(H)
    lc.n_sink = n_sink
    if n_sink:
        g = torch.Generator(device=DEV).manual_seed(3)
        lc.set_sinks(torch.randn((H, 128, n_sink), generator=g, device=DEV).half(),
                     torch.randn((H, n_sink, 128), generator=g, device=DEV).half())
    try:
        q = cu(O.rope_rotate_q(sp.q_vec(9), n_sink + L, theta))
        lc.precision = "fp32"
        want = lc.attend(q).clone()
        k, v = lc.dequantize(rope_theta=theta)
        if n_sink:
            k = torch.cat([lc.sink_k.transpose(1, 2), k], 1)
            v = torch.cat([lc.sink_v, v], 1)
        with sdpa_kernel(SDPBackend.MATH):
            got = torch.nn.functional.scaled_dot_product_attention(q[None, :, None], k[None].float(), v[None].float(),
                                                                   scale=1.0 / math.sqrt(128))[0, :, 0]
        assert rel_err(got.cpu().numpy(), want.cpu().numpy())[0] < 2e-3, rel_err(got.cpu().numpy(), want.cpu().numpy())
    finally:
        lc.sink_k = lc.sink_v = None
        lc.n_sink = 0


@gpu
def test_in_place_writes_touch_exactly_the_target_slice():
    bits, H, L = 3, 32, 1000
    c, lc = appended_cache(bits, H, L)
    S, at, start, stop = 1500, 211, 31, 700
    n = stop - start
    for rope in (None, 10000.0):
        kbuf = torch.full((H, S, 128), -1234.0, dtype=torch.float16, device=DEV)
        vbuf = torch.full((H, S, 128), 4321.0, dtype=torch.float16, device=DEV)
        k, v = lc.dequantize(start, stop, rope_theta=rope)
        rk, rv = lc.dequantize(start, stop, rope_theta=rope, out_k=kbuf[:, at:at + n], out_v=vbuf[:, at:at + n])
        assert rk.data_ptr() == kbuf[:, at:at + n].data_ptr() and rv.data_ptr() == vbuf[:, at:at + n].data_ptr()
        for buf, ref, fill in ((kbuf, k, -1234.0), (vbuf, v, 4321.0)):
            assert torch.equal(buf[:, at:at + n].view(torch.int16), ref.view(torch.int16))
            outside = torch.cat([buf[:, :at], buf[:, at + n:]], 1)
            assert bool((outside == fill).all())
    # caller outputs are validated before the launch
    with pytest.raises(ValueError):
        lc.dequantize(0, 10, out_k=kbuf[:, 1:11], out_v=vbuf[:, 1:11].transpose(0, 1).contiguous().transpose(0, 1))
    with pytest.raises(TypeError):
        lc.dequantize(0, 10, out_k=kbuf[:, :10].float(), out_v=vbuf[:, :10])
    with pytest.raises(ValueError):
        lc.dequantize(0, 10, out_k=kbuf[:, :9], out_v=vbuf[:, :9])
    with pytest.raises(ValueError):
        lc.dequantize(0, L + 1)
    with pytest.raises(ValueError):
        lc.dequantize(5, 4)
    lc.use_native_v = False
    try:
        with pytest.raises(NotImplementedError):
            lc.dequantize()
    finally:
        lc.use_native_v = True


@gpu
def test_empty_ranges_return_empty_outputs():
    from kvquant_b200 import _lib
    from kvquant_b200.cache import LayerCache
    bits, H = 4, 32
    klut, vcent = quantizer(bits, H)
    fresh = LayerCache.from_luts(bits, H, 64, klut, vcent, device=DEV)
    for lc, start, stop in ((fresh, 0, None), (appended_cache(bits, H, 1000)[1], 5, 5)):
        for rope in (None, 10000.0):
            n0 = _lib.launch_count()
            k, v = lc.dequantize(start, stop, rope_theta=rope)
            assert k.shape == v.shape == (H, 0, 128) and k.dtype == v.dtype == torch.float16
            buf = torch.zeros((H, 8, 128), dtype=torch.float16, device=DEV)
            rk, rv = lc.dequantize(start, stop, rope_theta=rope, out_k=buf[:, 3:3], out_v=buf[:, 8:])
            assert rk.shape == rv.shape == (H, 0, 128) and bool((buf == 0).all())
            assert _lib.launch_count() == n0


@gpu
def test_one_caller_output_and_separate_head_strides():
    """out_k and out_v may come from buffers of different lengths; an output not given is allocated."""
    bits, H, L = 4, 40, 1000
    c, lc = appended_cache(bits, H, L)
    start, stop = 100, 420
    n = stop - start
    k, v = lc.dequantize(start, stop, rope_theta=10000.0)
    kbuf = torch.full((H, 700, 128), 7.0, dtype=torch.float16, device=DEV)
    vbuf = torch.full((H, 333, 128), 7.0, dtype=torch.float16, device=DEV)
    rk, rv = lc.dequantize(start, stop, rope_theta=10000.0, out_k=kbuf[:, 50:50 + n])
    assert torch.equal(kbuf[:, 50:50 + n], k) and torch.equal(rv, v) and rv.is_contiguous()
    rk, rv = lc.dequantize(start, stop, rope_theta=10000.0, out_v=vbuf[:, 13:13 + n])
    assert torch.equal(vbuf[:, 13:13 + n], v) and torch.equal(rk, k)
    kbuf.fill_(7.0)
    lc.dequantize(start, stop, rope_theta=10000.0, out_k=kbuf[:, 1:1 + n], out_v=vbuf[:, :n])
    assert torch.equal(kbuf[:, 1:1 + n], k) and torch.equal(vbuf[:, :n], v)
    assert bool((kbuf[:, 0] == 7.0).all()) and bool((kbuf[:, 1 + n:] == 7.0).all())


@gpu
def test_dequantize_is_graph_capturable():
    """With caller outputs and an existing rope table, dequantize allocates nothing and captures into a CUDA graph;
    a replay reads the cache's current contents."""
    bits, H, L = 3, 32, 1000
    c, lc = appended_cache(bits, H, L)
    kbuf = torch.empty((H, L + 64, 128), dtype=torch.float16, device=DEV)
    vbuf = torch.empty_like(kbuf)
    ok, ov = kbuf[:, 64:], vbuf[:, 64:]
    for rope in (None, 10000.0):
        lc.dequantize(rope_theta=rope, out_k=ok, out_v=ov)           # eager warm-up (builds the rope table)
        torch.cuda.synchronize()
        want_k, want_v = ok.clone(), ov.clone()
        # no allocation by the call itself (counted eagerly: beginning a capture allocates torch's RNG state tensors)
        n_alloc = torch.cuda.memory_stats()["allocation.all.allocated"]
        lc.dequantize(rope_theta=rope, out_k=ok, out_v=ov)
        assert torch.cuda.memory_stats()["allocation.all.allocated"] == n_alloc
        s = torch.cuda.Stream()
        s.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(s):
            g = torch.cuda.CUDAGraph()
            with torch.cuda.graph(g, stream=s):
                lc.dequantize(rope_theta=rope, out_k=ok, out_v=ov)
        torch.cuda.current_stream().wait_stream(s)
        kbuf.zero_(); vbuf.zero_()
        g.replay()
        torch.cuda.synchronize()
        assert torch.equal(ok, want_k) and torch.equal(ov, want_v)
        assert bool((kbuf[:, :64] == 0).all()) and bool((vbuf[:, :64] == 0).all())
        saved = lc.vaff.clone()
        lc.vaff[:, 1] += 0.5                                          # V offsets moved: the replay sees it
        g.replay()
        torch.cuda.synchronize()
        lc.vaff.copy_(saved)
        assert torch.equal(ok, want_k) and not torch.equal(ov, want_v)
        lc.dequantize(rope_theta=rope, out_k=ok, out_v=ov)
        assert torch.equal(ov, want_v)
        del g


@gpu
def test_64_bit_output_offsets():
    """A dense-only 4-bit 32-head cache of 540K slots: 32 x 540K x 128 = 2.2e9 elements per output, past 2^31.  The
    last tokens (and a few earlier ones) against the oracle's dequantisation of the same words."""
    from kvquant_b200.cache import LayerCache
    bits, H, L = 4, 32, 540_000
    assert H * L * 128 > 2 ** 31
    klut, vcent = quantizer(bits, H)
    lc = LayerCache.from_luts(bits, H, L, klut, vcent, device=DEV, include_sparse=False)
    g = torch.Generator(device=DEV).manual_seed(5)
    for t in (lc.kcache, lc.vcache):
        t.copy_(torch.randint(-2 ** 31, 2 ** 31, t.shape, generator=g, device=DEV, dtype=torch.int64).to(torch.int32))
    lc.vaff[:, 0] = torch.rand(L, generator=g, device=DEV) + 0.5
    lc.vaff[:, 1] = torch.rand(L, generator=g, device=DEV) - 0.5
    lc.len = L
    k, v = lc.dequantize()
    tok = np.concatenate([np.arange(L - 64, L), [0, 1, 123_457, 524_287, 524_288]])
    ti = torch.as_tensor(tok, device=DEV)
    kw = lc.kcache[:, :, ti].cpu().numpy().reshape(-1, len(tok))
    vw = lc.vcache[:, :, ti].cpu().numpy().reshape(-1, len(tok))
    kk = O.k_dequant(kw, np.asarray(klut["lut"], np.float32), bits)
    assert np.array_equal(k[:, ti].cpu().numpy(), head_major(kk, H).astype(np.float16))
    aff = lc.vaff[ti].cpu().numpy().astype(np.float64)
    vv = lc.v_cent.cpu().numpy().astype(np.float64)[O.unpack_codes(vw, bits).astype(np.int64)] * aff[:, 0] + aff[:, 1]
    want = head_major(vv, H)
    d = np.abs(v[:, ti].cpu().numpy().astype(np.float64) - want.astype(np.float16).astype(np.float64))
    assert np.all(d <= fp16_ulp(want)), d.max()


def chunk_reference(c, lc, q, k, v, theta):
    """float64 causal attention of the chunk (q [T,H,128], k/v [T,hidden]) over sinks + the oracle's reconstruction of
    the cache (rotated) + the chunk's fp16 K (rotated) and V.  torch float64 on the device."""
    H, L, T = lc.H, lc.len, q.shape[0]
    ns = lc.n_sink if lc.sink_k is not None else 0
    p0 = lc.n_sink + lc.pos_base + L
    parts_k, parts_v = [], []
    if ns:
        parts_k.append(lc.sink_k.transpose(1, 2).double().cpu().numpy())
        parts_v.append(lc.sink_v.double().cpu().numpy())
    if L:
        parts_k.append(head_major(rotate_k(k_recon(c), np.arange(L) + lc.n_sink + lc.pos_base,
                                           theta), H))
        parts_v.append(head_major(v_recon(c), H))
    kr = rotate_k(k.T.astype(np.float64), np.arange(T) + p0, theta).astype(np.float16).astype(np.float64)
    parts_k.append(head_major(kr, H))
    parts_v.append(head_major(v.T.astype(np.float16).astype(np.float64), H))
    K = torch.from_numpy(np.concatenate(parts_k, 1)).to(DEV)      # [H, S, 128]
    V = torch.from_numpy(np.concatenate(parts_v, 1)).to(DEV)
    Q = torch.from_numpy(q.astype(np.float64)).to(DEV).transpose(0, 1)   # [H, T, 128]
    s = Q @ K.transpose(1, 2) / math.sqrt(128)
    S = K.shape[1]
    allowed = torch.arange(S, device=DEV)[None, :] <= (ns + L + torch.arange(T, device=DEV))[:, None]
    s = s.masked_fill(~allowed, float("-inf"))
    return (torch.softmax(s, -1) @ V).transpose(0, 1).cpu().numpy()   # [T, H, 128]


@gpu
@pytest.mark.parametrize("T", [1, 7, 64, 300])
@pytest.mark.parametrize("L", [0, 1000])
@pytest.mark.parametrize("n_sink", [0, 4])
def test_attend_chunk_against_float64(T, L, n_sink):
    """Tolerance 4e-3 of max |out|: q, K and V enter SDPA as fp16 (2^-11 = 4.9e-4 relative each); scaled scores here
    reach |s| ~ 10, so a score moves by up to ~5e-3 absolute, which moves the softmax-weighted output by a few 1e-3
    of its scale at worst, and the fp16 output adds another 2.4e-4 (measured errors sit near 1e-3)."""
    from kvquant_b200.cache import LayerCache
    bits, H, theta = 4, 32, 10000.0
    sp = spec(H)
    if L:
        c, lc = appended_cache(bits, H, L)
    else:
        klut, vcent = quantizer(bits, H)
        c = None
        lc = LayerCache.from_luts(bits, H, 64, klut, vcent, device=DEV)
    lc.n_sink = n_sink
    if n_sink:
        g = torch.Generator(device=DEV).manual_seed(4)
        lc.set_sinks(torch.randn((H, 128, n_sink), generator=g, device=DEV).half(),
                     torch.randn((H, n_sink, 128), generator=g, device=DEV).half())
    try:
        p0 = n_sink + L
        q = np.stack([O.rope_rotate_q(sp.q_vec(100 + i), p0 + i, theta) for i in range(T)])
        k, v = sp.k_tokens(T, seed=31 + T), sp.v_tokens(T, seed=32 + T)
        names = ("kcache", "vcache", "vaff", "vlut", "k_outliers", "k_outlier_idx", "v_outliers", "v_outlier_idx")
        before = {n: getattr(lc, n).clone() for n in names}
        got = lc.attend_chunk(cu(q), cu(k), cu(v), rope_theta=theta)
        assert got.shape == (T, H, 128) and got.dtype == torch.float32
        for n in names:
            assert torch.equal(getattr(lc, n), before[n]), n
        assert lc.len == L
        want = chunk_reference(c, lc, q, k, v, theta)
        assert rel_err(got.cpu().numpy(), want)[0] < 4e-3, rel_err(got.cpu().numpy(), want)
    finally:
        lc.sink_k = lc.sink_v = None
        lc.n_sink = 0


@gpu
def test_attend_chunk_of_one_token_equals_append_then_attend():
    """T = 1 is one decode step: attend_chunk over the cache == append the token, then attend (the appended token is
    quantised there, exact in the chunk, so the two agree to the quantisation error of one token out of 1001)."""
    bits, H, L, theta = 4, 32, 1000, 10000.0
    c, lc = appended_cache(bits, H, L)
    sp = spec(H)
    q = cu(O.rope_rotate_q(sp.q_vec(77), L, theta))
    k, v = cu(sp.k_tokens(1, seed=78)), cu(sp.v_tokens(1, seed=79))
    got = lc.attend_chunk(q[None], k, v, rope_theta=theta)[0]
    from kvquant_b200.cache import LayerCache
    lc2 = LayerCache.from_luts(bits, H, lc.Lmax, *quantizer(bits, H), device=DEV)
    lc2.load_state(c)
    lc2.append(k[0], v[0])
    lc2.precision = "fp32"
    want = lc2.attend(q)
    assert rel_err(got.cpu().numpy(), want.cpu().numpy())[0] < 1e-2
