"""Batched and paged decode at serving batch sizes: B up to 256 (the ABI's limit), where the launch geometry differs
from the B <= 8 of tests/test_gpu_batch.py and tests/test_gpu_paged.py.

Every kernel of the batched attend shares the SMs among the sequences, so as B grows each sequence is cut into fewer
token ranges, down to one CTA per head group walking the whole sequence (a V combine over one partial, a k_ratio CTA
whose last round has 1 to 15 live columns), and the grid takes more than one wave.  `launch_geometry` restates the
three launch formulas; each case takes B on both sides of every boundary it has (derived from the device's SM count)
and B = 256, and records the geometry it reached in its assertion messages.

* the batched attend against float64 per sequence (sinks, idle slots, lengths at the 16 / 80 / 240-token edges, one
  sequence at L_cap and one clamped to it, len_add 0 and 1), and call to call on dense caches;
* the paged attend (pages of 160 and 320, shuffled pool, lengths clamped by npages) against the contiguous batch --
  bit for bit on dense caches, within 8 fp32 ulps of each head's max with outlier rows -- and against float64 at 256;
* batched and paged appends at B = 67 and 256 against single caches (inactive and full slots, page crossings);
* one contiguous batch whose K / V slices start past 2^31 words;
* LLaMA-3.1 scaled rotary (k_outlier_pers_kernel with a frequency vector, one K range per sequence) against float64;
* a 2-layer LLaMA-3-8B BatchedDecoderStage graph at B = 67, contiguous and paged, against single-sequence runs;
* kvq_dec_rope_split_batch / _freq at B = 256 and at the grid-y limit 65535 against HF's rotation in float64.
The geometry helper is checked against hand-derived thresholds without a GPU.
"""
import numpy as np
import pytest
import torch

import test_gpu_batch as TB
import test_gpu_gqa as G
import test_gpu_paged as TP
import test_gpu_rope_scaling as R

gpu = pytest.mark.gpu
DEV = G.DEV


# ---- launch geometry ----------------------------------------------------------------------------------------------------
def _v_head_groups(bits, Hq, Hkv):
    """G of launch_vn (kvq_vnative.cu): 1 when the whole slab and its tables fit in 227 KiB with at least 2 ring
    stages (vn_stages over vn_smem_layout), else 2."""
    W, tabn, grp = 4 * bits, {4: 256, 3: 64, 2: 16}[bits], Hq // Hkv
    for groups in (1, 2):
        Hg = Hq // groups
        for S in (3, 2):
            off_w = (Hg // grp) * W * 32 * 4 * S + tabn * 256
            off_ws = (off_w + 2 * Hg * 33 * 4 + 15) & ~15
            if off_ws + 2 * Hg * 36 * 4 + 8 * 3 + 1024 <= 227 * 1024:
                return groups
    raise ValueError("no V layout fits")


def launch_geometry(bits, Hq, Hkv, B, sms):
    """Per-sequence launch geometry of the batched attend's kernels at batch size B on `sms` SMs:
    * dense K (launch_k_ratio, kvq_kratio.cu): CTA head groups of at most GMAX query heads (16 at 4 bits, 32
      otherwise) in whole KV groups; max_splits = sms / (groups * B), at least 1 -- the token ranges of a long sequence;
    * V (launch_vn, kvq_vnative.cu): ranges = max(1, sms / (G * B)), G head groups (_v_head_groups);
    * K outliers (k_outlier_grid, kvq_kscore.cu): max(1, sms * per_sm / B) persistent CTAs per sequence (the cap; fewer
      when L_cap * n_out / 512 is smaller), per_sm = 2 when the q table (Hq KiB) passes 56 KiB, else 4."""
    grp = Hq // Hkv
    kv_max = (16 if bits == 4 else 32) // grp
    k_groups = -(-Hkv // kv_max)
    v_groups = _v_head_groups(bits, Hq, Hkv)
    per_sm = 2 if Hq * 1024 > 56 * 1024 else 4
    return dict(B=B, k_groups=k_groups, k_splits=max(1, sms // (k_groups * B)), v_groups=v_groups,
                v_ranges=max(1, sms // (v_groups * B)), out_ctas=max(1, sms * per_sm // B))


def _last_multi(bits, Hq, Hkv, sms, key):
    """Last B in [1, 256] at which `key` is still >= 2 (None when it is 1 already at B = 1 or never reaches 1)."""
    multi = [B for B in range(1, 257) if launch_geometry(bits, Hq, Hkv, B, sms)[key] >= 2]
    return multi[-1] if multi and multi[-1] < 256 else None


def bracket(bits, Hq, Hkv, sms):
    """B values on both sides of the K, V and outlier boundaries (where they fall inside [1, 256]), and 256."""
    out = {256}
    for key in ("k_splits", "v_ranges", "out_ctas"):
        b = _last_multi(bits, Hq, Hkv, sms, key)
        if b is not None:
            out |= {b, b + 1}
    return sorted(out)


def _sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


def test_launch_geometry_thresholds_on_132_sms():
    # (bits, Hq, Hkv): K CTA groups, last B with >= 2 K ranges, V groups, last B with >= 2 V ranges, last B with >= 2
    # outlier CTAs (None: still >= 2 at B = 256) -- an H100 SXM's 132 SMs, worked out by hand from the launch code
    table = {(3, 32, 8): (1, 66, 1, 66, None), (4, 32, 8): (2, 33, 1, 66, None), (4, 32, 32): (2, 33, 1, 66, None),
             (2, 32, 32): (1, 66, 1, 66, None), (4, 40, 40): (3, 22, 2, 33, None), (4, 64, 8): (4, 16, 1, 66, 132)}
    for (bits, Hq, Hkv), (kg, kb, vg, vb, ob) in table.items():
        g = launch_geometry(bits, Hq, Hkv, 1, 132)
        assert (g["k_groups"], g["v_groups"]) == (kg, vg), (bits, Hq, Hkv, g)
        assert _last_multi(bits, Hq, Hkv, 132, "k_splits") == kb
        assert _last_multi(bits, Hq, Hkv, 132, "v_ranges") == vb
        assert _last_multi(bits, Hq, Hkv, 132, "out_ctas") == ob
        assert launch_geometry(bits, Hq, Hkv, kb + 1, 132)["k_splits"] == 1
        assert launch_geometry(bits, Hq, Hkv, vb + 1, 132)["v_ranges"] == 1
    assert bracket(4, 64, 8, 132) == [16, 17, 66, 67, 132, 133, 256]
    assert bracket(4, 40, 40, 132) == [22, 23, 33, 34, 256]
    assert bracket(3, 32, 8, 132) == [66, 67, 256]
    # V head groups: 2 from 4-bit MHA H = 36 and 3-bit MHA H = 60 on (the head-split V forms)
    assert [_v_head_groups(4, h, h) for h in (32, 36)] == [1, 2]
    assert [_v_head_groups(3, h, h) for h in (56, 60)] == [1, 2]
    assert _v_head_groups(2, 64, 64) == 1 and _v_head_groups(4, 64, 8) == 1


# ---- shared fixtures ----------------------------------------------------------------------------------------------------
EDGES = (0, 1, 15, 16, 17, 79, 80, 81, 239, 240, 241, 255, 256, 257, 1031, 1537, 2047)
L_CAP = 2100
LMAX = 2240            # a multiple of 160 and 320: the paged copies have the contiguous batch's Lmax


def _lengths(B, seed):
    """Per-sequence lengths cycling through EDGES from a seed-dependent start; the last sequence sits at L_CAP and the
    one before it holds 100 tokens more (its device length is clamped to L_CAP)."""
    lens = [EDGES[(b + seed) % len(EDGES)] for b in range(B)]
    if B >= 3:
        lens[-1], lens[-2] = L_CAP, L_CAP + 100
    return lens


def _set_sinks(caches, B, Hkv, n_sink, seed):
    g = torch.Generator(device=DEV).manual_seed(seed)
    sk = torch.randn((B, Hkv, 128, n_sink), generator=g, device=DEV).half()
    sv = torch.randn((B, Hkv, n_sink, 128), generator=g, device=DEV).half()
    for c in caches:
        c.set_sinks(sk, sv)


def _oracles(bc, q, lens, L_cap, oracle=None):
    """float64 (out, lse) of every sequence over min(lens[b], L_cap) tokens (the sinks alone at 0)."""
    want = []
    for b, n in enumerate(lens):
        lc = bc.seq(b)
        n = min(n, L_cap)
        if n == 0:
            want.append(TB._oracle_sinks(lc, q[b]))
            continue
        saved, lc.len = lc.len, n
        want.append(oracle(lc, q[b]) if oracle else G._oracle_gqa(lc, q[b]))
        lc.len = saved
    return want


def _check_all(out, lse, want, lens, what):
    for b, w in enumerate(want):
        G._check((out[b], lse[b]), w, "%s seq %d (L=%d)" % (what, b, lens[b]))


def _geometry(bits, Hq, Hkv, B):
    return launch_geometry(bits, Hq, Hkv, B, _sms())


# ---- 1. batched attend against float64 ----------------------------------------------------------------------------------
ATTEND_CASES = ((3, 32, 8, "kv"), (4, 32, 8, "k"), (4, 32, 32, "kv"), (2, 32, 32, "dense"), (4, 40, 40, "kv"),
                (4, 64, 8, "kv"))


def _attend_params():
    sms = _sms() if torch.cuda.is_available() else 132
    return [pytest.param(bits, Hq, Hkv, mode, B, id="%db-%d-%d-%s-B%d" % (bits, Hq, Hkv, mode, B))
            for bits, Hq, Hkv, mode in ATTEND_CASES for B in bracket(bits, Hq, Hkv, sms)]


@gpu
@pytest.mark.parametrize("bits,Hq,Hkv,mode,B", _attend_params())
def test_batched_attend_at_scale_against_float64(bits, Hq, Hkv, mode, B):
    geo = _geometry(bits, Hq, Hkv, B)
    lens = _lengths(B, seed=bits + Hq + B)
    bc = TB._batch(bits, Hq, Hkv, B, mode, Lmax=LMAX, n_sink=3)
    _set_sinks([bc], B, Hkv, 3, seed=B)
    TB._fill(bc, lens, 1000 + B)
    q = TB._queries(bc, 17 + B)
    want = _oracles(bc, q, lens, L_CAP)
    out, lse = TB._battend(bc, q, L_cap=L_CAP)
    _check_all(out, lse, want, lens, "len_add=0 %s" % geo)
    if mode == "dense":   # a fixed summation order: call to call bit for bit
        again = TB._battend(bc, q, L_cap=L_CAP)
        assert torch.equal(again[0], out) and torch.equal(again[1], lse), geo
    # the decode step's form: device lengths one lower and len_add = 1 (an idle slot at -1 + 1 = 0)
    bc.lens -= 1
    out1 = torch.full_like(out, float("nan"))
    lse1 = torch.full_like(lse, float("nan"))
    bc.attend(q, out=out1, lse=lse1, L_cap=L_CAP, len_add=1)
    torch.cuda.synchronize()
    _check_all(out1, lse1, want, lens, "len_add=1 %s" % geo)
    if mode == "dense":
        assert torch.equal(out1, out) and torch.equal(lse1, lse), geo


# ---- 2. paged attend ----------------------------------------------------------------------------------------------------
def _paged_params():
    sms = _sms() if torch.cuda.is_available() else 132
    return [pytest.param(bits, Hq, Hkv, B, id="%db-%d-%d-B%d" % (bits, Hq, Hkv, B))
            for bits, Hq, Hkv in ((3, 32, 8), (4, 40, 40)) for B in bracket(bits, Hq, Hkv, sms)]


@gpu
@pytest.mark.parametrize("bits,Hq,Hkv,B", _paged_params())
def test_paged_attend_at_scale(bits, Hq, Hkv, B):
    """Pages of 160 and 320 over shuffled pools, every fifth sequence of 1000+ tokens with two pages fewer mapped than
    its length needs (clamped); dense and K+V outlier caches."""
    geo = _geometry(bits, Hq, Hkv, B)
    lens = _lengths(B, seed=B)
    for mode in ("dense", "kv"):
        bc = TB._batch(bits, Hq, Hkv, B, mode, Lmax=LMAX, n_sink=2)
        TB._fill(bc, lens, 3000 + B)
        q = TB._queries(bc, 40 + B)
        for P in (160, 320):
            n_pool = sum(-(-n // P) for n in lens) + 7
            pc = TP._paged(bits, Hq, Hkv, B, P, n_pool, LMAX // P, mode, n_sink=2, seed=B + P)
            TP._load(pc, bc, lens)
            _set_sinks([bc, pc], B, Hkv, 2, seed=P)
            eff = list(lens)
            for b in range(0, B, 5):
                if lens[b] >= 1000:
                    k = -(-lens[b] // P) - 2
                    pc.pages.npages[b] = k
                    eff[b] = k * P
            assert eff != lens
            bc.lens.copy_(torch.tensor(eff, dtype=torch.int64))
            what = "%s P=%d %s" % (mode, P, geo)
            out, lse = TP._pattend(pc, q, L_cap=LMAX)
            o1, l1 = TB._battend(bc, q, L_cap=LMAX)
            if mode == "dense":
                assert torch.equal(out, o1) and torch.equal(lse, l1), what
                again = TP._pattend(pc, q, L_cap=LMAX)
                assert torch.equal(again[0], out) and torch.equal(again[1], lse), what
            else:
                assert TB._close(out, o1), what
                live = torch.isfinite(l1)
                assert torch.equal(torch.isfinite(lse), live), what
                assert float((lse - l1)[live].abs().max()) < 1e-6 * float(l1[live].abs().max() + 1), what
            if B == 256 and mode == "kv":
                _check_all(out, lse, _oracles(bc, q, eff, LMAX), eff, what)
            bc.lens.copy_(torch.tensor(lens, dtype=torch.int64))


# ---- 3. batched and paged appends ---------------------------------------------------------------------------------------
@gpu
@pytest.mark.parametrize("bits", (3, 4))
@pytest.mark.parametrize("B", (67, 256))
def test_batched_and_paged_appends_at_scale(bits, B):
    """After a prefill at mixed lengths (around the 160-token page edges) and 4 batched appends with every third slot
    inactive and some slots full (479 fills then drops, 480 drops): every tensor of every sequence is bit-identical to
    single caches given the same tokens, and the paged copy (pages of 160, 3 per slot) reads back as the batch."""
    from kvquant_b200.cache import LayerCache
    Hq, Hkv, Lmax, P, steps = 32, 8, 480, 160, 4
    geo = _geometry(bits, Hq, Hkv, B)
    _, klut, vcent = G._calibration(bits, Hkv)
    bc = TB._batch(bits, Hq, Hkv, B, "kv", Lmax=Lmax)
    singles = [LayerCache.from_luts(bits, Hkv, Lmax, klut, vcent, device=DEV, include_sparse=True, sparse_v=True,
                                    q_heads=Hq) for _ in range(B)]
    for t in [bc.kcache, bc.vcache] + [c.kcache for c in singles] + [c.vcache for c in singles]:
        t.fill_(0x5A5A5A5A)    # a stray write shows
    edges = (0, 1, 157, 158, 159, 160, 161, 317, 318, 319, 320, 321, 250, 400, 479, 480)
    start = [edges[(5 * b) % len(edges)] for b in range(B)]
    for b, n in enumerate(start):
        if n:
            k, v = G._tokens(singles[b], n, 7000 + b)
            bc.seq(b).append_chunk(k, v)
            singles[b].append_chunk(k, v)
    bc.commit()
    pc = TP._paged(bits, Hq, Hkv, B, P, n_pool=3 * B + 5, max_pages=3, mode="kv", seed=bits)
    TP._load(pc, bc, start)
    lens = list(start)
    active = torch.tensor([int(b % 3 != 2) for b in range(B)], dtype=torch.int32, device=DEV)
    act = active.tolist()
    for step in range(steps):
        for b in range(B):
            if act[b]:
                pc.pages.reserve(b, min(lens[b] + 1, pc.pages.cap))
        k, v = G._tokens(singles[0], B, 8000 + step)
        bc.append_dyn(k, v, active=active)
        bc.advance(active=active)
        pc.append_dyn(k, v, active=active)
        pc.advance(active=active)
        for b in range(B):
            if act[b]:
                if lens[b] < Lmax:
                    singles[b].append_dyn(k[b], v[b], torch.tensor([lens[b]], dtype=torch.int64, device=DEV))
                lens[b] += 1
    torch.cuda.synchronize()
    assert bc.lens.tolist() == lens == pc.lens.tolist(), geo
    for b in range(B):
        s = singles[b]
        for name in TP._tensors(s):
            assert torch.equal(getattr(bc, name)[b], getattr(s, name)), (name, b, B)
        n = min(lens[b], Lmax)
        pc.pages.lens_host[b] = n
        lc = TP._single(bits, Hq, Hkv, Lmax, "kv")
        pc.read_seq(b, lc)
        assert lc.len == n
        TP._same_slots(lc, s, n)


# ---- 4. offsets past 2^31 words -----------------------------------------------------------------------------------------
@gpu
def test_sequence_slices_past_2_31_words():
    """A contiguous batch of B = 256 sequences, 4 bits, Hkv = 8 (Hq = 32), Lmax = 69632: each sequence's K and V slice is
    8 * 16 * 69632 = 8,912,896 words, so sequences 241-255 start past 2^31 words in the two packed cache tensors.  Only
    the cache tensors pass 2^31 elements; the V LUT, (sf, off) and outlier rows stay below it, so this case does not
    cover 64-bit offsets into those.  Sequences 0, 1, 241 and 255 hold about 2000 tokens (append_chunk on the views
    and batched appends); the others are idle.  The appended state equals single caches given the same tokens, nothing
    is written anywhere else, and the attend matches float64."""
    from kvquant_b200.cache import n_outliers_each
    bits, Hq, Hkv, B, Lmax, L_cap = 4, 32, 8, 256, 69632, 2100
    W = 4 * bits
    per_seq = Hkv * W * Lmax
    assert 240 * per_seq < 2 ** 31 <= 241 * per_seq and B * per_seq > 2 ** 31
    n_out = 2 * n_outliers_each(Hkv * 128, 0.99)
    need = B * Lmax * (2 * Hkv * W * 4 + (2 ** bits) * 4 + 2 * 4 + 2 * n_out * 8)   # K, V, vlut, vaff, K / V outliers
    assert B * Lmax * n_out < 2 ** 31 and B * Lmax * 2 ** bits < 2 ** 31
    free, _ = torch.cuda.mem_get_info()
    if free < need + (2 << 30):
        pytest.skip("needs %.1f GB of device memory for the caches (+2 GB), %.1f GB free" % (need / 1e9, free / 1e9))
    from kvquant_b200.cache import LayerCache
    _, klut, vcent = G._calibration(bits, Hkv)
    bc = TB._batch(bits, Hq, Hkv, B, "kv", Lmax=Lmax)
    live = (0, 1, 241, 255)
    singles = {b: LayerCache.from_luts(bits, Hkv, 2112, klut, vcent, device=DEV, include_sparse=True, sparse_v=True,
                                       q_heads=Hq) for b in live}
    active = torch.zeros(B, dtype=torch.int32, device=DEV)
    active[list(live)] = 1

    def chunk(sizes, seed):
        for b, n in zip(live, sizes):
            k, v = G._tokens(singles[b], n, seed + b)
            bc.seq(b).append_chunk(k, v)
            singles[b].append_chunk(k, v)
        bc.commit()

    def steps(n, seed):
        for i in range(n):
            k, v = G._tokens(singles[0], B, seed + i)
            bc.append_dyn(k, v, active=active)
            bc.advance(active=active)
            for b in live:
                singles[b].append_dyn(k[b], v[b], torch.tensor([singles[b].len], dtype=torch.int64, device=DEV))
                singles[b].len += 1
        bc.sync_host()

    chunk((1990, 1931, 1999, 1957), 100)
    steps(3, 200)
    chunk((7, 64, 1, 30), 300)
    steps(3, 400)
    torch.cuda.synchronize()
    for b in live:
        s, n = singles[b], singles[b].len
        assert bc.seq(b).len == n
        for name in ("kcache", "vcache"):
            assert torch.equal(getattr(bc, name)[b][..., :n], getattr(s, name)[..., :n]), (name, b)
            assert not bool(getattr(bc, name)[b][..., n:].any()), (name, b)
        for name in ("vlut", "vaff", "k_outliers", "k_outlier_idx", "v_outliers", "v_outlier_idx"):
            assert torch.equal(getattr(bc, name)[b][:n], getattr(s, name)[:n]), (name, b)
    for b in range(B):
        if b not in live:
            for name in ("kcache", "vcache", "vaff", "k_outliers", "v_outliers"):
                assert not bool(getattr(bc, name)[b].any()), (name, b)
    q = TB._queries(bc, 5)
    out, lse = TB._battend(bc, q, L_cap=L_cap)
    for b in range(B):
        if b in live:
            G._check((out[b], lse[b]), G._oracle_gqa(bc.seq(b), q[b]), "seq %d" % b)
        else:
            assert torch.equal(out[b], torch.zeros_like(out[b])) and bool(torch.isneginf(lse[b]).all()), b


# ---- 5. scaled rotary ---------------------------------------------------------------------------------------------------
@gpu
@pytest.mark.parametrize("paged", (False, True))
def test_llama31_rotary_at_scale(paged):
    """LLaMA-3.1 rotary at B = 67, 3 bits, 32/8, K+V outliers: the batched (and paged) k_outlier_pers_kernel with a
    frequency vector, one K range per sequence on a 132-SM H100, against float64 from HF's fp32 angles."""
    spec = R.LLAMA31
    bits, Hq, Hkv, B, Lmax = 3, 32, 8, 67, 1120
    geo = _geometry(bits, Hq, Hkv, B)
    lens = [min(n, 1100) for n in _lengths(B, seed=5)]
    lens[-2] = 1120        # past L_cap = 1100: clamped
    bc = TB._batch(bits, Hq, Hkv, B, "kv", Lmax=Lmax, n_sink=2)
    TB._fill(bc, lens, 500)
    cache = bc
    if paged:
        cache = TP._paged(bits, Hq, Hkv, B, 160, sum(-(-n // 160) for n in lens) + 3, Lmax // 160, "kv", n_sink=2,
                          seed=9)
        TP._load(cache, bc, lens)
    _set_sinks([bc, cache], B, Hkv, 2, seed=6)
    q = torch.stack([R.rotate_q(spec, G._query(Hq, 300 + b), 2 + min(n, 1100)) for b, n in enumerate(lens)])
    out = torch.full((B, Hq, 128), float("nan"), device=DEV)
    lse = torch.full((B, Hq), float("nan"), device=DEV)
    cache.attend(q, out=out, lse=lse, L_cap=1100, rope=spec)
    torch.cuda.synchronize()
    want = _oracles(bc, q, lens, 1100, oracle=lambda lc, qb: R.oracle(lc, qb, spec))
    _check_all(out, lse, want, lens, "paged=%s %s" % (paged, geo))


# ---- 6. the graph step --------------------------------------------------------------------------------------------------
@gpu
def test_batched_stage_graph_at_b67_matches_single_sequences():
    """A 2-layer LLaMA-3-8B-shaped BatchedDecoderStage at B = 67, contiguous and paged (a pool of 280 pages of 160
    tokens, less than B x max_len), prompts of 1 to 500 tokens, every third slot inactive, 6 graph replays with slot 1
    retired and refilled after the third.  Every active slot's logits follow a fresh single-sequence run (prefill +
    forward_torch) within 1e-2 of their max; inactive slots keep their lengths."""
    from kvquant_b200 import decode as kd
    st, _ = TB._stage("llama3_8b")
    cfg = st.cfg
    B, N, refill = 67, 6, 3
    gen = torch.Generator().manual_seed(23)
    plens = [int(x) for x in torch.randint(1, 501, (B,), generator=gen)]
    plens[:3] = [500, 1, 160]
    prompts = [torch.randint(0, cfg.vocab, (n,), generator=gen).to(DEV) for n in plens]
    new_prompt = torch.randint(0, cfg.vocab, (321,), generator=gen).to(DEV)
    toks = torch.randint(0, cfg.vocab, (N, B), generator=gen)
    act = [b % 3 != 2 for b in range(B)]

    def run(paged):
        bst = kd.BatchedDecoderStage(st, B, page_size=160, n_pool=280) if paged else kd.BatchedDecoderStage(st, B)
        if paged:
            assert bst.pages.n_pool * bst.pages.P < B * cfg.max_len
        for b in range(B):
            bst.set_active(b, act[b])
        for b, p in enumerate(prompts):
            bst.prefill_seq(b, st.embed[p], chunk=256)
        g = kd.BatchedGraphedStep(bst)
        got = []
        for i in range(N):
            if i == refill:
                bst.reset_seq(1)
                bst.prefill_seq(1, st.embed[new_prompt], chunk=256)
            g.tok.copy_(toks[i].to(DEV))
            g.replay()
            torch.cuda.synchronize()
            got.append(g.logits.float().clone())
        want_lens = [n + N * a for n, a in zip(plens, act)]
        want_lens[1] = new_prompt.shape[0] + N - refill
        assert bst.lens.tolist() == want_lens, paged
        return got

    runs = {paged: run(paged) for paged in (False, True)}
    for b in range(B):
        if not act[b]:
            continue
        if b == 1:
            ref = (TB._single_reference(st, prompts[1], toks[:refill, 1].tolist())
                   + TB._single_reference(st, new_prompt, toks[refill:, 1].tolist()))
        else:
            ref = TB._single_reference(st, prompts[b], toks[:, b].tolist())
        for paged, got in runs.items():
            for i in range(N):
                assert torch.isfinite(got[i][b]).all(), (paged, b, i)
                d = (ref[i] - got[i][b]).abs().max().item()
                assert d <= 1e-2 * max(1.0, ref[i].abs().max().item()), (paged, b, i, d)


# ---- 7. the batched rotary split ----------------------------------------------------------------------------------------
@gpu
@pytest.mark.parametrize("rope", ("theta", "llama3", "yarn"))
@pytest.mark.parametrize("Hq,Hkv,B", ((32, 8, 256), (4, 4, 65535)))
def test_rope_split_batch_at_its_limits(Hq, Hkv, B, rope):
    """kvq_dec_rope_split_batch (theta 500000) and kvq_dec_rope_split_freq (LLaMA-3.1, YaRN: attention factor != 1) at
    B = 256 and at the grid-y limit 65535, row b at position pos[b] + 3 with positions up to 2^20: the query against HF's
    apply_rotary_pos_emb in float64 from the fp32 angle f_j * p (a few fp32 ulps of |q|), K and V copied exactly."""
    from kvquant_b200 import _lib
    lib = _lib.load()
    n = (Hq + 2 * Hkv) * 128
    g = torch.Generator(device=DEV).manual_seed(B)
    qkv = torch.randn((B, n), generator=g, device=DEV).half()
    pos = torch.randint(0, 1 << 20, (B,), generator=g, device=DEV, dtype=torch.int64)
    pos[:4] = torch.tensor([0, 65533, 65534, (1 << 20) - 4])
    if rope == "theta":
        inv = (1.0 / (500000.0 ** (torch.arange(0, 128, 2, dtype=torch.float32) / 128))).to(DEV)
        attn = 1.0
    else:
        spec = R.SPECS[rope]
        inv, attn = spec.inv_freq.float().to(DEV), float(spec.attention_factor)
    q, k, v = (torch.full((B, m), float("nan"), device=DEV) for m in (Hq * 128, Hkv * 128, Hkv * 128))
    if rope == "theta":
        rc = lib.kvq_dec_rope_split_batch(qkv.data_ptr(), inv.data_ptr(), pos.data_ptr(), 3, q.data_ptr(),
                                          k.data_ptr(), v.data_ptr(), Hq, Hkv, B, None)
    else:
        rc = lib.kvq_dec_rope_split_freq(qkv.data_ptr(), inv.data_ptr(), attn, pos.data_ptr(), 3, q.data_ptr(),
                                         k.data_ptr(), v.data_ptr(), Hq, Hkv, B, None)
    _lib.check(rc)
    torch.cuda.synchronize()
    hq = Hq * 128
    assert torch.equal(k, qkv[:, hq:hq + Hkv * 128].float()) and torch.equal(v, qkv[:, hq + Hkv * 128:].float())
    f = inv.cpu().numpy()
    for r0 in range(0, B, 8192):
        rows = slice(r0, min(B, r0 + 8192))
        p = (pos[rows].cpu().numpy() + 3).astype(np.float32)
        ang = (f[None, :] * p[:, None]).astype(np.float32).astype(np.float64)        # [rows, 64]: HF's fp32 angle
        c = np.concatenate([np.cos(ang), np.cos(ang)], 1)[:, None, :] * attn
        s = np.concatenate([np.sin(ang), np.sin(ang)], 1)[:, None, :] * attn
        x = qkv[rows, :hq].double().cpu().numpy().reshape(-1, Hq, 128)
        rot = np.concatenate([-x[..., 64:], x[..., :64]], -1)
        want = x * c + rot * s
        got = q[rows].double().cpu().numpy().reshape(-1, Hq, 128)
        bound = 2.0 ** -21 * attn * (np.abs(x) + np.abs(rot))
        err = np.abs(got - want) - bound
        assert (err <= 0).all(), (r0, float(err.max()), np.argwhere(err > 0)[:4].tolist())
