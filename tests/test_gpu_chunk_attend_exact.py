"""kvq_attend_chunk / LayerCache.attend_chunk_fused pinned by exact probes instead of a tolerance.

The kernel is deterministic (no atomics on the result path, a fixed combine order), and with q = 0 every softmax
weight is exactly 1.0 in fp16.  So most of what can go wrong in its tile walk -- a key dropped or doubled at a tile,
split or query-block edge, a read past the cached length, a head mixed up with another -- is checkable bit for bit
or to a few fp32 ulps, where the float64 comparison of test_gpu_attend_chunk_fused.py (1.8e-3 of each head's max)
cannot see it.

CPU: the key-split bookkeeping over SM counts 1..300, every head count and T, L up to 2^20.
GPU, on caches whose state the tests write directly:
  counting probe   q = 0 and integer V: out[i, h, c] is the mean of the V values row i may see, within 4 fp32 ulps;
  poisoned inputs  NaN / random words past the cached length, outside the rope columns in use and in the split
                   scratch leave the output bit-identical;
  head isolation   NaN in one head's LUT rows, sinks, q, chunk K/V or outlier entries reaches that head only;
  peaked softmax   one key 90 nats above the rest, on every tile and split edge, rising maxima, a split whose
                   combine weight underflows: the output is that key's V (or the mean of the rest) to fp32 rounding;
  outlier budgets  n_each = 1, 21, 41, 64 (n_out = 128 at 4 heads) through the counting probe and float64.
Every split count and split edge comes from the device's SM count through the restated rule n_splits."""
import math

import numpy as np
import pytest
import torch

from _util import quantizer, spec
from test_gpu_attend_chunk_fused import (BK, BQ, MAX_SMS, MAX_SPLITS, TOL, chunk_inputs, head_err, n_splits,
                                         reference, set_sinks, split_starts)

DEV = "cuda:0"
gpu = pytest.mark.gpu
PAD = 64                 # rows past Lmax that every synthetic cache owns: a read past the allocation lands there
ULPS = 4                 # exact probes: the sums are exact, the result is one division (two roundings, one split)


def split_plan(T, H, L, sms):
    """(split count, slot tiles per split) as the launcher picks them (kvq_chunk.cu launch)."""
    n = n_splits(T, H, L, sms)
    tiles = -(-L // BK)
    return n, (-(-tiles // n) if n > 1 else max(tiles, 1))


# ---------------------------------------------------------------------------------------------------------------------
# CPU: split bookkeeping
# ---------------------------------------------------------------------------------------------------------------------
SWEEP_T = [1, 2, 63, 64, 65, 127, 128, 129, 255, 256, 257, 1000, 4095, 4096, 4097, 65536, 65537, 1 << 20]
SWEEP_L = [0, 1, 2, 63, 64, 65, 127, 128, 129, 191, 192, 193, 2047, 2048, 2049, 2111, 2113, 4096, 4097, 65536,
           65537, (1 << 20) - 1, 1 << 20]


def test_split_bookkeeping_on_every_device_and_shape():
    """For SM counts 1..300, H = 4..64 and T, L over the tile edges up to 2^20: the split count the launcher picks is
    1..32, uses no more CTAs than SMs when above 1, puts every slot tile in exactly one split (the kernel's
    s0 = min(s * per, tiles), n_slot = min(s0 + per, tiles) - s0) with no split empty, and the scratch size the host
    allocates covers its partials."""
    from kvquant_b200 import _lib
    lib = _lib.load()
    seen = set()
    for H in range(4, 65, 4):
        for T in SWEEP_T:
            base = -(-T // BQ) * H
            for L in SWEEP_L:
                tiles = -(-L // BK)
                plans = {split_plan(T, H, L, sms) for sms in range(1, 301)}
                scratch = lib.kvq_attend_chunk_scratch_bytes(H, T, L)
                for n, per in plans:
                    assert 1 <= n <= MAX_SPLITS, (H, T, L, n)
                    if n > 1:
                        assert n * base <= MAX_SMS and tiles >= 2, (H, T, L, n)
                        assert scratch >= n * T * H * 130 * 4, (H, T, L, n, scratch)
                    if tiles:
                        assert (n - 1) * per < tiles <= n * per, (H, T, L, n, per)   # no split empty, none missed
                    seen.add((tiles, n, per))
    # the kernel's own per-split arithmetic, tile by tile, for every distinct plan met above
    for tiles, n, per in seen:
        hits = np.zeros(max(tiles, 1), dtype=np.int64)
        for s in range(n):
            s0 = min(s * per, tiles)
            n_slot = min(s0 + per, tiles) - s0
            assert n_slot >= 1 or tiles == 0, (tiles, n, per, s)
            hits[s0:s0 + n_slot] += 1
        assert tiles == 0 or np.all(hits == 1), (tiles, n, per)
    assert max(n for _, n, _ in seen) == MAX_SPLITS and len({n for _, n, _ in seen}) > 20


def test_split_plan_matches_the_counts_the_gpu_tests_rely_on():
    """The restated plan at a few hand-checked points (the device's own split count is read back from the scratch
    by test_scratch_poison_and_the_device_split_count)."""
    assert split_plan(130, 4, 4000, 132) == (16, 4) and split_plan(1, 4, 4000, 132) == (32, 2)
    assert split_plan(1, 4, 2049, 132) == (17, 2) and split_plan(1, 4, 2048, 132) == (32, 1)
    assert split_plan(2100, 4, 4000, 132) == (1, 63) and split_plan(1, 64, 0, 132) == (1, 1)
    assert split_plan(1, 4, 1000, 1) == (1, 16) and split_plan(1, 4, 1000, 1000) == (16, 1)


# ---------------------------------------------------------------------------------------------------------------------
# GPU helpers: caches written directly, integer value encodings, the direct C call
# ---------------------------------------------------------------------------------------------------------------------
def synth_cache(bits, H, Lmax, mode="kv", threshold=0.99, seed=0):
    """LayerCache of Lmax slots holding random state: packed words, a K LUT N(0, 1), (sf, off), and outlier rows with
    distinct indices spread over every head.  Every buffer is a view into an allocation PAD rows longer (lc.pads),
    so the tests can poison memory just past the cache without any pointer leaving what they own."""
    from kvquant_b200.cache import LayerCache
    g = torch.Generator(device=DEV).manual_seed(seed)
    hid, nl = H * 128, 2 ** bits
    klut = torch.randn((hid, nl), generator=g, device=DEV)
    thr = torch.zeros((hid, nl - 1), device=DEV)
    vcent = torch.randn(nl, generator=g, device=DEV).sort().values
    lc = LayerCache(bits, H, Lmax, klut, None, thr, thr, vcent, DEV, include_sparse=mode != "dense",
                    sparsity_threshold=threshold, sparse_v=mode == "kv")
    W = 128 * bits // 32
    lc.pads = {}
    for name in ("kcache", "vcache"):
        buf = torch.randint(-2 ** 31, 2 ** 31, (H * W * Lmax + PAD * W,), generator=g, device=DEV,
                            dtype=torch.int64).to(torch.int32)
        setattr(lc, name, buf[:H * W * Lmax].view(H, W, Lmax))
        lc.pads[name] = buf
    vaff = torch.empty((Lmax + PAD, 2), device=DEV)
    vaff[:, 0] = torch.rand(Lmax + PAD, generator=g, device=DEV) + 0.5
    vaff[:, 1] = torch.rand(Lmax + PAD, generator=g, device=DEV) - 0.5
    lc.vaff, lc.pads["vaff"] = vaff[:Lmax], vaff
    for side, on in (("k", lc.sparse_k), ("v", lc.sparse_v)):
        if on:
            val = torch.randn((Lmax + PAD, lc.n_out), generator=g, device=DEV)
            idx = torch.rand((Lmax + PAD, hid), generator=g, device=DEV).argsort(1)[:, :lc.n_out]
            idx = idx.to(torch.int32).contiguous()
            setattr(lc, side + "_outliers", val[:Lmax])
            setattr(lc, side + "_outlier_idx", idx[:Lmax])
            lc.pads[side + "_outliers"], lc.pads[side + "_outlier_idx"] = val, idx
    lc.len = Lmax
    return lc


def ihash(key, h, c, salt):
    """A small integer in [-30, 30] per (key, head, channel), broadcast over the three index tensors: neighbouring keys,
    heads and channels get unrelated values, and each salt is an unrelated encoding."""
    x = (key * 73856093) ^ (h * 19349663) ^ (c * 83492791) ^ (salt * 2654435761)
    return (x % 61 - 30).double()


def ar(n):
    return torch.arange(n, device=DEV, dtype=torch.int64)


def set_integer_values(lc, ns, salt, T):
    """V of every key an integer: sinks and chunk ihash per (key, head, channel); slot t (all Lmax of them, so a slot
    past the length that leaks in is counted) (sf, off) = (0, ihash) plus integer V outliers.  Sinks get random K.
    Returns (chunk v f32 [T, hidden], V of [sinks | slots 0..Lmax-1] float64 [H, ns + Lmax, 128])."""
    H, hid = lc.H, lc.hidden
    hh, cc = ar(H)[:, None, None], ar(128)[None, None, :]
    g = torch.Generator(device=DEV).manual_seed(salt)
    lc.n_sink, lc.pos_base = ns, 0
    if ns:
        lc.set_sinks(torch.randn((H, 128, ns), generator=g, device=DEV).half(),
                     ihash(ar(ns)[None, :, None], hh, cc, salt).half())
    else:
        lc.sink_k = lc.sink_v = None
    off = ihash(ns + ar(lc.Lmax), H, 0, salt)
    lc.vaff[:, 0] = 0.0
    lc.vaff[:, 1] = off.float()
    slot_v = off[None, :, None].expand(H, lc.Lmax, 128).clone()
    if lc.sparse_v:
        vals = ihash(ar(lc.Lmax)[:, None], H + 1, ar(lc.n_out)[None, :], salt)
        lc.v_outliers.copy_(vals)
        add = torch.zeros((lc.Lmax, hid), dtype=torch.float64, device=DEV)
        add.scatter_add_(1, lc.v_outlier_idx.long(), vals)
        slot_v += add.view(lc.Lmax, H, 128).transpose(0, 1)
    v = ihash(ns + lc.Lmax + ar(T)[:, None, None], ar(H)[None, :, None], ar(128)[None, None, :], salt)
    parts = [slot_v] if not ns else [lc.sink_v.double(), slot_v]
    return v.view(T, hid).float(), torch.cat(parts, 1)


def mean_of_visible(V_sl, ns, L, v, T):
    """float64 [T, H, 128]: row i averages the V of sinks, slots 0..L-1 and chunk tokens 0..i (prefix sums)."""
    H = V_sl.shape[0]
    Vall = torch.cat([V_sl[:, :ns + L], v.double().view(T, H, 128).transpose(0, 1)], 1)
    cs = Vall.cumsum(1)[:, ns + L:]
    return (cs / (ns + L + 1 + ar(T)).double()[None, :, None]).transpose(0, 1)


def fp32_ulps(got, want, floor=0.0):
    """max over elements of |got - want| in fp32 ulps of want (float64); differences up to `floor` count as 0."""
    w = want.float().abs()
    ulp = (torch.nextafter(w, torch.full_like(w, math.inf)) - w).double()
    d = ((got.double() - want).abs() - floor).clamp_min(0)
    return float((d / ulp).max())


def counting_probe(lc, ns, L, T, salt, values=None):
    """q = 0: out[i] must be the mean of the visible V to ULPS fp32 ulps (a key dropped or doubled anywhere moves
    it by about 1/(ns + L + i) of a value, thousands of ulps).  `values`: what set_integer_values(lc, ns, salt, T')
    returned for some T' >= T (the cache is left as it wrote it).  Returns the ulps seen."""
    lc.len = L
    v, V_sl = set_integer_values(lc, ns, salt, T) if values is None else values
    v = v[:T]
    q = torch.zeros((T, lc.H, 128), device=DEV)
    k = torch.randn((T, lc.hidden), device=DEV)
    got = lc.attend_chunk_fused(q, k, v)
    e = fp32_ulps(got, mean_of_visible(V_sl, ns, L, v, T))
    assert e <= ULPS, (lc.bits, lc.H, ns, L, T, salt, e)
    return e


def call_chunk(lc, q, kc, vc, rope, npos, pos0, out, scratch, L=None):
    """The C entry point with every operand given: the chunk's fp16 K/V, the rope table and the scratch included."""
    from kvquant_b200 import _lib
    L = lc.len if L is None else L
    ns = lc.n_sink if lc.sink_k is not None else 0
    _lib.check(lc.lib.kvq_attend_chunk(
        lc.bits, lc.H, lc.Lmax, L, q.shape[0], q.data_ptr(), kc.data_ptr(), vc.data_ptr(),
        lc.kcache.data_ptr(), lc.klut_deq.data_ptr(), *lc._out_ptrs("k"),
        lc.vcache.data_ptr(), lc.v_cent_deq.data_ptr(), lc.vaff.data_ptr(), *lc._out_ptrs("v"),
        lc.n_out, rope.data_ptr(), npos, pos0, lc.sink_k.data_ptr() if ns else None,
        lc.sink_v.data_ptr() if ns else None, ns, out.data_ptr(), scratch.data_ptr(),
        torch.cuda.current_stream().cuda_stream), "kvq_attend_chunk")
    return out


def chunk16(lc, k, v, theta, p0):
    kc = torch.empty((lc.H, k.shape[0], 128), dtype=torch.float16, device=DEV)
    vc = torch.empty_like(kc)
    lc._chunk_kv16(k, v, theta, p0, kc, vc)
    return kc, vc


def bits_of(x):
    return x.contiguous().view(torch.int32)


def sms():
    return torch.cuda.get_device_properties(DEV).multi_processor_count


def split_change_lengths(T, H, Lmax, keep=6):
    """Lengths L <= Lmax at which the split count changes (and L - 1): the first, the last and a few between."""
    s = sms()
    ch = [L for L in range(1, Lmax + 1) if n_splits(T, H, L, s) != n_splits(T, H, L - 1, s)]
    pick = ch if len(ch) <= keep else [ch[int(round(i * (len(ch) - 1) / (keep - 1)))] for i in range(keep)]
    return sorted({x for L in pick for x in (L - 1, L)})


# ---------------------------------------------------------------------------------------------------------------------
# GPU: counting probe
# ---------------------------------------------------------------------------------------------------------------------
@gpu
@pytest.mark.parametrize("bits", [4, 3, 2])
def test_counting_probe_at_every_head_count(bits):
    for H in range(4, 65, 4):
        lc = synth_cache(bits, H, 1088, seed=H)
        for salt in (1, 2):
            for ns, L, T in ((65, 1000, 130), (0, 129, 1)):
                counting_probe(lc, ns, L, T, salt)


GRID_T = [1, 15, 16, 17, 63, 64, 65, 127, 128, 129, 255, 256, 257, 2048]
GRID_L = [0, 1, 63, 64, 65, 127, 128, 129]
GRID_NS = [0, 1, 63, 64, 65, 128, 130]


@gpu
@pytest.mark.parametrize("H", [4, 24, 64])
def test_counting_probe_over_the_edge_grid(H):
    """Every T edge of the query blocks, every L edge of the slot tiles plus the lengths where the split count changes
    (derived from the device's SM count), every sink-tile edge up to a third sink tile, two encodings."""
    Lmax = 2176
    lc = synth_cache(4, H, Lmax, seed=100 + H)
    splits = set()
    lengths = {T: sorted(set(GRID_L) | set(split_change_lengths(T, H, 2112))) for T in GRID_T}
    for salt in (1, 2):
        for ns in GRID_NS:
            values = set_integer_values(lc, ns, salt, max(GRID_T))
            for T in GRID_T:
                for L in lengths[T]:
                    splits.add(n_splits(T, H, L, sms()))
                    counting_probe(lc, ns, L, T, salt, values)
    assert len(splits) >= (3 if H < 64 else 1), splits


@gpu
def test_counting_probe_at_a_long_chunk():
    """T = 8192 (64 query blocks) after 64 sinks and 1000 slots: every row, both encodings."""
    lc = synth_cache(4, 4, 1088, seed=5)
    for salt in (1, 2):
        counting_probe(lc, 64, 1000, 8192, salt)


@gpu
@pytest.mark.parametrize("mode", ["dense", "k_only", "kv"])
@pytest.mark.parametrize("H", [4, 32])
def test_counting_probe_in_every_cache_form(mode, H):
    lc = synth_cache(3, H, 1088, mode=mode, seed=7)
    for T in (1, 129, 300):
        for L in (0, 65, 1000):
            for ns in (0, 65):
                for salt in (1, 2):
                    counting_probe(lc, ns, L, T, salt)


# ---------------------------------------------------------------------------------------------------------------------
# GPU: poisoned inputs leave the output bit-identical
# ---------------------------------------------------------------------------------------------------------------------
@gpu
@pytest.mark.parametrize("H,T", [(4, 130), (32, 17)])
@pytest.mark.parametrize("L", [1, 65, 1000, 1088])
def test_nothing_past_the_length_is_read(H, T, L):
    """NaN in (sf, off) and in the K and V outlier values of every slot >= L (their indices pointing at every head),
    random words in the packed K and V past L -- up to PAD rows past the allocation when L == Lmax -- and the output
    does not move by one bit."""
    lc = synth_cache(4, H, 1088, seed=L)
    set_sinks(lc, 5)
    lc.len = L
    q, k, v = chunk_inputs(H, T, seed=L)
    clean = lc.attend_chunk_fused(q, k, v)
    assert torch.isfinite(clean).all()
    g = torch.Generator(device=DEV).manual_seed(L + 1)
    P = lc.pads
    P["vaff"][L:] = float("nan")
    for side in ("k", "v"):
        P[side + "_outliers"][L:] = float("nan")
        P[side + "_outlier_idx"][L:] = torch.randint(0, H * 128, P[side + "_outlier_idx"][L:].shape, generator=g,
                                                     device=DEV, dtype=torch.int32)
    for name in ("kcache", "vcache"):
        words = torch.randint(-2 ** 31, 2 ** 31, P[name].shape, generator=g, device=DEV,
                              dtype=torch.int64).to(torch.int32)
        getattr(lc, name)[:, :, L:] = words[:getattr(lc, name)[:, :, L:].numel()].view_as(getattr(lc, name)[:, :, L:])
        P[name][getattr(lc, name).numel():] = words[getattr(lc, name).numel():]
    got = lc.attend_chunk_fused(q, k, v)
    assert torch.equal(bits_of(got), bits_of(clean))


@gpu
@pytest.mark.parametrize("H,T", [(4, 130), (32, 129)])
@pytest.mark.parametrize("pos0", [0, 70_000])
def test_rope_columns_outside_the_slots_are_not_read(H, T, pos0):
    """The C entry point with a rope table that is NaN outside columns [pos0, pos0 + L), and a larger npos than the
    clean table's: bit-identical output.  The chunk's fp16 K/V come from the clean table beforehand."""
    from kvquant_b200 import quant_cuda as qc
    L, theta = 1000, 10000.0
    lc = synth_cache(4, H, 1088, seed=3)
    set_sinks(lc, 5)
    lc.len = L
    q, k, v = chunk_inputs(H, T, seed=9)
    clean, _, npos = qc.rope_tables(lc.device, theta, pos0 + L + T)
    kc, vc = chunk16(lc, k, v, theta, pos0 + L)
    scratch = torch.zeros(max(lc.lib.kvq_attend_chunk_scratch_bytes(H, T, L), 16), dtype=torch.uint8, device=DEV)
    a = call_chunk(lc, q, kc, vc, clean, npos, pos0, torch.empty((T, H, 128), device=DEV), scratch)
    npos_p = pos0 + L + T + 300
    poisoned = torch.full((64, npos_p, 2), float("nan"), device=DEV)
    poisoned[:, pos0:pos0 + L] = clean[:, pos0:pos0 + L]
    b = call_chunk(lc, q, kc, vc, poisoned, npos_p, pos0, torch.empty((T, H, 128), device=DEV), scratch)
    assert torch.isfinite(a).all()
    assert torch.equal(bits_of(a), bits_of(b))


@gpu
@pytest.mark.parametrize("H,T,L", [(4, 130, 1000), (4, 1, 4000), (8, 300, 700)])
def test_scratch_poison_and_the_device_split_count(H, T, L):
    """Scratch filled with 0xFF bytes (NaN) before a call with several key splits: bit-identical output to a call on
    a zeroed scratch.  Afterwards exactly the partials of the restated split count are written -- nsplit x T x H
    rows of 130 floats, all finite -- and the rest is still 0xFF: the device split the keys as the rule says."""
    lc = synth_cache(4, H, 4032, seed=11)
    set_sinks(lc, 5)
    lc.len = L
    n = n_splits(T, H, L, sms())
    assert n > 1, n
    q, k, v = chunk_inputs(H, T, seed=12)
    kc, vc = chunk16(lc, k, v, 10000.0, 5 + L)
    from kvquant_b200 import quant_cuda as qc
    rope, _, npos = qc.rope_tables(lc.device, 10000.0, 5 + L + T)
    size = lc.lib.kvq_attend_chunk_scratch_bytes(H, T, L)
    zero = torch.zeros(size, dtype=torch.uint8, device=DEV)
    ff = torch.full((size,), 0xFF, dtype=torch.uint8, device=DEV)
    a = call_chunk(lc, q, kc, vc, rope, npos, 5, torch.empty((T, H, 128), device=DEV), zero)
    b = call_chunk(lc, q, kc, vc, rope, npos, 5, torch.empty((T, H, 128), device=DEV), ff)
    assert torch.isfinite(a).all()
    assert torch.equal(bits_of(a), bits_of(b))
    part = ff.view(torch.float32)
    used = n * T * H * 130
    assert torch.isfinite(part[:used]).all()
    assert torch.equal(ff[used * 4:], torch.full_like(ff[used * 4:], 0xFF))


# ---------------------------------------------------------------------------------------------------------------------
# GPU: head isolation
# ---------------------------------------------------------------------------------------------------------------------
POISONS = ["klut", "sink_k", "sink_v", "q", "chunk_k", "chunk_v", "k_out", "v_out"]


@gpu
@pytest.mark.parametrize("H,T,L", [(8, 130, 1000), (64, 64, 300)])
def test_a_poisoned_head_reaches_no_other_head(H, T, L):
    """NaN in head g's K LUT rows, sink K, sink V, q, chunk K or chunk V channels, or as the value of the K / V
    outlier entries whose index lies in head g: every query row of head g becomes non-finite and every other head is
    bit-identical to the clean call.  At 8 heads a slot's outlier row holds entries of several heads and the keys are
    split (on an H100); at 64 heads one split.  Poisoned tensors are cloned and restored."""
    lc = synth_cache(4, H, 1088, seed=H)
    set_sinks(lc, 5)
    lc.len = L
    q, k, v = chunk_inputs(H, T, seed=13)
    clean = lc.attend_chunk_fused(q, k, v)
    assert torch.isfinite(clean).all()
    if H == 8:
        assert n_splits(T, H, L, sms()) > 1
        owners = (lc.k_outlier_idx[:L] >> 7)
        assert all(len(owners[t].unique()) >= 4 for t in (0, L - 1))
    nan = float("nan")
    for g in (0, H // 2 + 1, H - 1):
        for what in POISONS:
            q2, k2, v2 = q, k, v
            saved = None
            hs = slice(g * 128, (g + 1) * 128)
            if what == "klut":
                saved = (lc.klut_deq, lc.klut_deq.clone())
                lc.klut_deq[hs] = nan
            elif what in ("sink_k", "sink_v"):
                t = getattr(lc, what)
                saved = (t, t.clone())
                t[g] = nan
            elif what == "q":
                q2 = q.clone()
                q2[:, g] = nan
            elif what == "chunk_k":
                k2 = k.clone()
                k2[:, hs] = nan
            elif what == "chunk_v":
                v2 = v.clone()
                v2[:, hs] = nan
            else:
                val, idx = (lc.k_outliers, lc.k_outlier_idx) if what == "k_out" else (lc.v_outliers, lc.v_outlier_idx)
                saved = (val, val.clone())
                val[(idx >> 7) == g] = nan
            try:
                got = lc.attend_chunk_fused(q2, k2, v2)
            finally:
                if saved is not None:
                    saved[0].copy_(saved[1])
            assert (~torch.isfinite(got[:, g])).any(-1).all(), (g, what)
            others = [h for h in range(H) if h != g]
            assert torch.equal(bits_of(got[:, others]), bits_of(clean[:, others])), (g, what)
    assert torch.equal(bits_of(lc.attend_chunk_fused(q, k, v)), bits_of(clean))      # everything restored


# ---------------------------------------------------------------------------------------------------------------------
# GPU: peaked softmax
# ---------------------------------------------------------------------------------------------------------------------
AMP_Q, AMP_K = 16.0, 64.0       # q and marked-key amplitudes: score 16 * 64 / sqrt(128) = 90.5 nats, all others 0
THETA = 1e6                     # channels 60..63 turn by < 0.01 rad over the 4260 positions used: scores along a
                                # rising pattern stay what their amplitudes say
RIVAL = 30.0                    # a rival key this many nats below the marked one: weight e^-30 against 1
FLOOR = 1e-10                   # absolute slack against the float64 softmax: the rival's weight leaves < 60 x e^-30
                                # = 6e-12 in its output, and its own rounding ~1e-16 where an output is exactly 0
                                # (where fp32 ulps are meaningless); every value here is a multiple of 1/4260


class Peaked:
    """H = 4 heads, 130 sinks (three sink tiles), L slots, T = 130 rows (two query blocks).  Every slot's K is 0 (zero
    K LUT, zero outlier values), so is every sink and chunk key, and q of head h is AMP_Q times the unit vector on
    channels (c_h, c_h + 64) rotated at a chosen position.  A key is marked by giving it K = amplitude x the same unit
    vector at its own position: a K outlier entry on channel c_h (slots), the sink's K, or the chunk token's
    pre-RoPE key.  V is the integer encoding of the counting probe, so every output is a plain mean or one V.
    channels=[0] * H: the fastest-turning channel (1 rad per position), so a slot rotated at a neighbour's position
    loses 37 of its 90.5 nats."""
    H, NS, T = 4, 130, 130

    def __init__(self, L=4000, T=130, channels=None):
        self.L, self.T = L, T
        self.lc = lc = synth_cache(4, self.H, 4032, mode="kv", seed=21)
        self.v, _ = set_integer_values(lc, self.NS, 3, T)
        lc.len = L
        lc.klut_deq.zero_()
        lc.k_outliers.zero_()
        lc.sink_k.zero_()
        self.ch = channels or [60 + h for h in range(self.H)]
        # entries 0..H-1 of every row: head h's channel c_h (the random others keep value 0)
        lc.k_outlier_idx[:, :self.H] = torch.tensor([h * 128 + c for h, c in enumerate(self.ch)], dtype=torch.int32,
                                                    device=DEV)
        from kvquant_b200 import quant_cuda as qc
        self.rope = qc.rope_tables(lc.device, THETA, self.NS + L + T + 1)[0]
        self.p_slot0 = self.NS          # rope position of slot 0 (n_sink + pos_base)
        self.k = torch.zeros((T, lc.hidden), device=DEV)

    def unit(self, pos):
        """[H, 128]: (cos, sin) of channel c_h at `pos` on channels (c_h, c_h + 64)."""
        u = torch.zeros((self.H, 128), device=DEV)
        for h, c in enumerate(self.ch):
            u[h, c], u[h, c + 64] = self.rope[c, pos, 0], self.rope[c, pos, 1]
        return u

    def aim(self, pos):
        return (AMP_Q * self.unit(pos)).half().float()[None].expand(self.T, self.H, 128).contiguous()

    def mark(self, kind, j, amp=AMP_K):
        """Give key j of a region K = amp x unit at its position; returns that position."""
        lc = self.lc
        if kind == "sink":
            lc.sink_k[:, :, j] = (amp * self.unit(0)).half()
            return 0
        if kind == "slot":
            lc.k_outliers[j, :self.H] = amp
            return self.p_slot0 + j
        for h, c in enumerate(self.ch):
            self.k[j, h * 128 + c] = amp
        return self.p_slot0 + self.L + j

    def rival(self, pos):
        """The last sink aimed where q is, RIVAL nats below a marked key: a marked slot that is not rotated at its own
        position falls below it."""
        f = 1.0 - RIVAL / (AMP_Q * AMP_K / math.sqrt(128))
        self.lc.sink_k[:, :, self.NS - 1] = (f * AMP_K * self.unit(pos)).half()

    def clear(self):
        self.lc.sink_k.zero_()
        self.lc.k_outliers.zero_()
        self.k.zero_()

    def marked_v(self, kind, j):
        lc = self.lc
        if kind == "sink":
            return lc.sink_v[:, j].double()
        if kind == "chunk":
            return self.v.view(self.T, self.H, 128)[j].double()
        _, V = lc.dequantize(j, j + 1)
        return V[:, 0].double()

    def run(self, q):
        got = self.lc.attend_chunk_fused(q, self.k, self.v, rope_theta=THETA)
        want = reference(self.lc, q, self.k, self.v, THETA)
        assert torch.isfinite(got).all()
        return got, want


def assert_fp32_exact(got, want, what):
    # the marked key's weight is 1, a rival's e^-30 and every other weight e^-90 or less: in fp16 they are all 0
    e = fp32_ulps(got, want, floor=FLOOR)
    assert e <= ULPS, (what, e)


@gpu
def test_a_marked_key_on_every_tile_and_split_edge_is_the_output():
    """The marked key on sink 0, 63, 64 and the last sink; slot 0, 63, 64, L-1 and the first and last slot of every
    key split (with a rival sink 30 nats below); chunk token 0 and the diagonal at rows 127 and 128.  Rows that see
    it output its V; the others the mean of what they see; both to ULPS fp32 ulps of a float64 attention over the
    same operands."""
    P = Peaked(channels=[0] * Peaked.H)
    lc, L, T = P.lc, P.L, P.T
    starts = split_starts(T, P.H, L, sms())
    assert len(starts) > 1 and len(starts) == n_splits(T, P.H, L, sms())
    ends = [s - 1 for s in starts[1:]] + [L - 1]
    marks = [("sink", j) for j in (0, 63, 64, P.NS - 1)] + \
            [("slot", j) for j in sorted({0, 63, 64, L - 1, *starts, *ends})] + \
            [("chunk", j) for j in (0, 127, 128)]
    for kind, j in marks:
        P.clear()
        pos = P.mark(kind, j)
        if kind == "slot":
            P.rival(pos)
        q = P.aim(pos)
        got, want = P.run(q)
        assert_fp32_exact(got, want, (kind, j))
        first = j if kind == "chunk" else 0
        mv = P.marked_v(kind, j)
        assert_fp32_exact(got[first:], mv[None].expand(T - first, -1, -1), (kind, j, "is the marked V"))
        if first:
            assert fp32_ulps(got[:first], want[:first], floor=FLOOR) <= ULPS, (kind, j)


@gpu
@pytest.mark.parametrize("T", [130, 2100])
def test_a_maximum_rising_in_every_tile_ends_in_the_last_tile_of_the_last_split(T):
    """Slot tile t holds one key 70 (t + 1) nats above 0: every tile of every split rescales its running sums by
    e^-70, and the last tile of the last split holds the maximum, whose V every row must output.  T = 130: several
    splits on an H100; T = 2100: one."""
    P = Peaked(T=T)
    L = P.L
    tiles = -(-L // BK)
    top = None
    for t in range(tiles):
        j = min(t * BK + (t * 23) % BK, L - 1)
        P.mark("slot", j, amp=70.0 * (t + 1) * math.sqrt(128) / AMP_Q)
        top = j
    q = P.aim(P.mark("slot", top, amp=70.0 * tiles * math.sqrt(128) / AMP_Q))
    got, want = P.run(q)
    assert_fp32_exact(got, want, T)
    assert_fp32_exact(got, P.marked_v("slot", top)[None].expand(T, -1, -1), (T, "is the top V"))


@gpu
@pytest.mark.parametrize("which", ["second", "last"])
def test_a_split_200_nats_below_the_rest_drops_out_of_the_combine(which):
    """Every slot of one key split (not split 0, which also holds the sinks and the chunk) scores -200 nats, every
    other key 0: that split's combine weight 2^(m_s - M) underflows to 0, and each row outputs the plain mean of the
    other keys it sees, finite and to ULPS ulps of float64."""
    P = Peaked()
    L, T = P.L, P.T
    starts = split_starts(T, P.H, L, sms())
    assert len(starts) > 2
    s = 1 if which == "second" else len(starts) - 1
    lo, hi = starts[s], (starts[s + 1] if s + 1 < len(starts) else L)
    P.lc.k_outliers[lo:hi, :P.H] = -200.0 * math.sqrt(128) / AMP_Q
    q = P.aim(P.p_slot0 + (lo + hi) // 2)
    got, want = P.run(q)
    assert fp32_ulps(got, want, floor=FLOOR) <= ULPS, which
    # the dropped split's keys are really out: the mean over the others differs from the mean over all
    allm = P.lc.attend_chunk_fused(torch.zeros_like(q), P.k, P.v, rope_theta=THETA)
    assert (got - allm).abs().max().item() > 1e-3


# ---------------------------------------------------------------------------------------------------------------------
# GPU: outlier budgets
# ---------------------------------------------------------------------------------------------------------------------
# (bits, H, sparsity_threshold, n_each): n_each = int((1 - threshold) / 2 * hidden) + 1, n_out = 2 n_each <= 128
BUDGETS = [(4, 32, 0.9999, 1), (3, 32, 0.99, 21), (4, 32, 0.98, 41), (2, 32, 0.969, 64), (4, 4, 0.752, 64)]


@gpu
@pytest.mark.parametrize("bits,H,threshold,n_each", BUDGETS)
def test_counting_probe_at_other_outlier_budgets(bits, H, threshold, n_each):
    for mode in ("kv", "k_only"):
        lc = synth_cache(bits, H, 1088, mode=mode, threshold=threshold, seed=n_each)
        assert lc.n_each == n_each and lc.n_out == 2 * n_each
        for salt in (1, 2):
            for ns, L, T in ((5, 1000, 130), (0, 1000, 1), (64, 65, 257)):
                counting_probe(lc, ns, L, T, salt)


@gpu
@pytest.mark.parametrize("bits,H,threshold,n_each", BUDGETS)
def test_against_float64_at_other_outlier_budgets(bits, H, threshold, n_each):
    """Caches filled by append_chunk at each outlier budget, against the float64 attention over the kernel's operands
    at test_gpu_attend_chunk_fused.py's tolerance."""
    from kvquant_b200.cache import LayerCache
    lc = LayerCache.from_luts(bits, H, 1088, *quantizer(bits, H), device=DEV, sparsity_threshold=threshold)
    assert lc.n_each == n_each
    sp = spec(H)
    k0 = torch.from_numpy(sp.k_tokens(1000, seed=21)).to(DEV)
    v0 = torch.from_numpy(sp.v_tokens(1000, seed=22)).to(DEV)
    for s0 in range(0, 1000, 500):
        lc.append_chunk(k0[s0:s0 + 500], v0[s0:s0 + 500])
    set_sinks(lc, 5)
    assert bool((lc.k_outliers[:1000] != 0).any()) and bool((lc.v_outliers[:1000] != 0).any())
    for i, (T, L) in enumerate([(1, 1000), (BQ + 1, 1000), (1, 129), (300, 700)]):
        lc.len = L
        q, k, v = chunk_inputs(H, T, seed=50 + i)
        err = head_err(lc.attend_chunk_fused(q, k, v), reference(lc, q, k, v, 10000.0))
        assert err < TOL, (T, L, err)
