"""Ragged prefill (DESIGN.md section 4.15): several slots' prompt chunks appended and attended in one launch
(kvq_append_kv_fused_chunk_ragged[_paged], kvq_attend_chunk_ragged[_paged]; BatchedLayerCache / PagedLayerCache
append_chunks and attend_chunks) and BatchedDecoderStage.prefill_seqs.

* ragged append: every named slot is bit for bit what per-slot append_chunk leaves (bits 2/3/4, kv / k / dense, heads
  32/32, 32/8, 64/8, 16/2, 8/1; contiguous, and paged with pages of 160 and 320 handed out shuffled); segment lengths
  1, 7, 8, 9, 300 and 0, start lengths that are not multiples of 8, slots in arbitrary order; slots not named and free
  pages are byte-unchanged;
* ragged attend: each segment's rows equal the lone attend_chunk_fused on its slot bit for bit (paged: on a read_seq
  copy), with sinks, a static RotarySpec, an empty slot and a slot whose lone call splits its keys, and lie within the
  chunk attends' float64 tolerance;
* stage: prefill_seqs of mixed prompts (empty slots, a follow-up after graph replays, a fork suffix, a prompt longer
  than `chunk`) against the prefill_seq loop, and the graph continues without recapture;
* refusals: duplicate slots, the cap, an exhausted pool, a shared page and length-dependent rotary change nothing.
"""
import numpy as np
import pytest
import torch

import test_gpu_batch as TB
import test_gpu_gqa as G
import test_gpu_paged as TP
import test_gpu_paged_prefill as PP

gpu = pytest.mark.gpu
DEV = G.DEV
THETA = G.THETA


def _snapshot(c):
    return {name: getattr(c, name).clone() for name in TP._tensors(c)}


def _equal(a, b):
    return all(torch.equal(a[k].view(torch.int32), b[k].view(torch.int32)) for k in a)


# ---- ragged append ---------------------------------------------------------------------------------------------------
STARTS = (0, 77, 160, 317, 5, 3)          # slot 5 is never named
ROUNDS = (((3, 300), (0, 9), (2, 1), (1, 0), (4, 7)),      # (slot, T) in call order
          ((1, 8), (4, 300), (0, 7), (3, 9), (2, 0)))


@gpu
@pytest.mark.parametrize("bits", (2, 3, 4))
@pytest.mark.parametrize("mode", ("kv", "k", "dense"))
@pytest.mark.parametrize("shape", ((32, 32), (32, 8), (64, 8), (16, 2), (8, 1)))
def test_ragged_append_is_bit_identical_to_per_slot_appends(bits, mode, shape):
    Hq, Hkv = shape
    P = 320 if bits == 3 else 160
    Lmax, B = 960, len(STARTS)
    bc = TB._batch(bits, Hq, Hkv, B, mode, Lmax=Lmax)
    pc = TP._paged(bits, Hq, Hkv, B, P, n_pool=B * (Lmax // P) + 3, max_pages=Lmax // P, mode=mode, seed=bits + Hkv)
    TP._poison(pc, range(pc.n_pool), 3)
    refs = []
    for b, n in enumerate(STARTS):
        lc = TP._single(bits, Hq, Hkv, Lmax, mode)
        if n:
            k, v = G._tokens(lc, n, 10 + b)
            lc.append_chunk(k, v)
            bc.seq(b).append_chunk(k, v)
        pc.load_seq(b, lc)
        refs.append(lc)
    bc.commit()
    pc.commit()
    for r, rnd in enumerate(ROUNDS):
        slots, counts = [b for b, _ in rnd], [t for _, t in rnd]
        k, v = G._tokens(refs[0], sum(counts), 100 + r)
        row = 0
        for b, t in rnd:
            refs[b].append_chunk(k[row:row + t], v[row:row + t])
            row += t
        untouched = _snapshot(bc.seq(5))
        held = set(p for b in range(B) for p in pc.pages.pages[b])
        free_before = _snapshot(pc)
        bc.append_chunks(slots, k, v, counts)
        pc.append_chunks(slots, k, v, counts)
        torch.cuda.synchronize()
        assert _equal(untouched, _snapshot(bc.seq(5)))
        free = [p for p in range(pc.n_pool) if p not in held and p not in set(q for b in range(B) for q in pc.pages.pages[b])]
        assert PP._pages_equal(pc, free_before, free)
        for b in range(B):
            assert bc.seq(b).len == refs[b].len == pc.lens_host[b]
            TP._same_slots(bc.seq(b), refs[b], refs[b].len)
            got = TP._single(bits, Hq, Hkv, Lmax, mode)
            pc.read_seq(b, got)
            TP._same_slots(got, refs[b], refs[b].len)
    assert bc.lens.tolist() == list(STARTS)     # host lengths only: commit publishes them


# ---- ragged attend ---------------------------------------------------------------------------------------------------
def _lone(lc, q, k, v, rope):
    return lc.attend_chunk_fused(q, k, v, rope_theta=THETA, rope=rope)


@gpu
@pytest.mark.parametrize("bits", (2, 3, 4))
@pytest.mark.parametrize("shape", ((32, 32), (32, 8), (16, 2), (8, 1)))
@pytest.mark.parametrize("rope", ("theta", "llama31"))
def test_ragged_attend_is_bit_identical_to_lone_calls(bits, shape, rope):
    from kvquant_b200.rope import RotarySpec
    Hq, Hkv = shape
    spec = None if rope == "theta" else RotarySpec(500000.0, {
        "rope_type": "llama3", "factor": 8.0, "low_freq_factor": 1.0, "high_freq_factor": 4.0,
        "original_max_position_embeddings": 8192})
    lens = (0, 317, 2000, 161)          # slot 2's lone call (50 rows over 2000 tokens) splits its keys on 132 SMs
    bc, pc, Lmax = TP._pair(bits, Hq, Hkv, lens, 320 if bits == 2 else 160, "kv", n_sink=5, extra=3, seed=bits)
    rnd = ((2, 50), (0, 131), (3, 0), (1, 260))
    slots, counts = [b for b, _ in rnd], [t for _, t in rnd]
    N = sum(counts)
    lc0 = bc.seq(0)
    q, k, v = G._chunk_inputs(lc0, N, seed=bits + Hkv)
    got_c = bc.attend_chunks(slots, q, k, v, counts, rope_theta=THETA, rope=spec)
    got_p = pc.attend_chunks(slots, q, k, v, counts, rope_theta=THETA, rope=spec)
    torch.cuda.synchronize()
    row = 0
    for b, t in rnd:
        if t == 0:
            continue
        sl = slice(row, row + t)
        want = _lone(bc.seq(b), q[sl].contiguous(), k[sl].contiguous(), v[sl].contiguous(), spec)
        assert torch.equal(got_c[sl], want), (b, "contiguous")
        paged_copy = G._cache(bits, Hq, Hkv, "kv", Lmax=Lmax, n_sink=5)
        pc.read_seq(b, paged_copy)
        paged_copy.set_sinks(pc.sink_k[b], pc.sink_v[b])
        want_p = _lone(paged_copy, q[sl].contiguous(), k[sl].contiguous(), v[sl].contiguous(), spec)
        assert torch.equal(got_p[sl], want_p), (b, "paged")
        if spec is None:
            assert G._chunk_err(got_c[sl], G._chunk_oracle(bc.seq(b), q[sl], k[sl], v[sl])) <= G.CHUNK_TOL, b
        row += t
    assert bc.lens_host == list(lens) and pc.lens_host == list(lens)   # the caches are not modified


# ---- stage -----------------------------------------------------------------------------------------------------------
def _logits_close(a, b, tol):
    return ((a - b).abs().max() / b.abs().max()).item() <= tol


# fp16 tolerance of stage outputs and logits between the two routes: prefill_seq attends through SDPA over a dequantised
# copy and prefill_seqs through the fused ragged attend, and the packed GEMMs have other shapes, so fp16 roundings differ
STAGE_TOL = 2e-2


@gpu
@pytest.mark.parametrize("paged", (False, True))
def test_prefill_seqs_follows_the_prefill_seq_loop(paged):
    """Two identical llama3_8b-shaped stages of B = 4.  History: slot 0 a 300-token prompt, slot 2 forked from it (paged)
    or given the same prompt (contiguous), three graph replays, then one prefill_seqs of a 97-token follow-up for slot
    0, a 140-token suffix for slot 2, a 700-token prompt for empty slot 1 (longer than chunk = 256, so rounds hold
    different segment sets) with slot 3 left alone; against prefill_seq of the same prompts one by one.  Outputs and
    the next replays' logits agree within STAGE_TOL, the seeded next-token argmax agrees, lengths and the untouched
    slot match, and the same graph keeps serving."""
    from kvquant_b200 import decode as kd
    st, _ = TB._stage("llama3_8b")
    cfg = st.cfg
    gen = torch.Generator().manual_seed(5)
    rnd = lambda n: torch.randint(0, cfg.vocab, (n,), generator=gen).to(DEV)   # noqa: E731
    p0, p3, follow0, suffix2, prompt1 = rnd(300), rnd(20), rnd(97), rnd(140), rnd(700)
    toks = torch.randint(0, cfg.vocab, (6, 4), generator=gen)
    runs = []
    for ragged in (False, True):
        bst = kd.BatchedDecoderStage(st, 4, page_size=160 if paged else None, n_pool=24 if paged else None)
        if paged:
            bst.pages._free = [int(p) for p in np.random.default_rng(1).permutation(bst.pages.n_pool)]
        bst.prefill_seq(0, st.embed[p0], chunk=256)
        if paged:
            bst.fork_seq(0, 2)
        else:
            bst.prefill_seq(2, st.embed[p0], chunk=256)
        bst.prefill_seq(3, st.embed[p3], chunk=256)
        bst.set_active(1, False)        # slot 1 stays empty until its prompt
        g = kd.BatchedGraphedStep(bst)
        for i in range(3):
            g.tok.copy_(toks[i].to(DEV))
            g.replay()
        torch.cuda.synchronize()
        if not paged:
            for bc in bst.caches:
                bc.sync_host()
        slot3 = [_snapshot(bc.seq(3)) for bc in bst.caches] if not paged else None
        before_src = [_snapshot(pc) for pc in bst.caches] if paged else None
        prompts = {0: st.embed[follow0], 2: st.embed[suffix2], 1: st.embed[prompt1]}
        if ragged:
            ys = bst.prefill_seqs(prompts, chunk=256, max_tokens=512)
        else:
            ys = {b: bst.prefill_seq(b, x, chunk=256) for b, x in prompts.items()}
        bst.set_active(1, True)
        torch.cuda.synchronize()
        assert bst.lens.tolist() == [400, 700, 443, 23]
        if paged:
            assert bst.pages.lens_host == [400, 700, 443, 23]
            for pc, snap in zip(bst.caches, before_src):    # slot 0's shared pages are byte-unchanged
                shared = [p for p in bst.pages.pages[0] if bst.pages.refs[p] > 1]
                assert shared and PP._pages_equal(pc, snap, shared)
        else:
            assert all(bc.lens_host == [400, 700, 443, 23] for bc in bst.caches)
            for bc, snap in zip(bst.caches, slot3):
                assert _equal(snap, _snapshot(bc.seq(3)))
        logits = []
        for i in range(3, 6):
            g.tok.copy_(toks[i].to(DEV))
            g.replay()
            torch.cuda.synchronize()
            logits.append(g.logits.float().clone())
        assert bst.lens.tolist() == [403, 703, 446, 26]
        runs.append((ys, logits))
    (y_ref, l_ref), (y_new, l_new) = runs
    for b in y_ref:
        assert y_new[b].shape == y_ref[b].shape
        assert _logits_close(y_new[b].float(), y_ref[b].float(), STAGE_TOL), b
    for a, b in zip(l_new, l_ref):
        assert _logits_close(a, b, STAGE_TOL)
        top = b.topk(2, dim=-1)
        clear = (top.values[:, 0] - top.values[:, 1]) > 2 * (a - b).abs().amax(dim=-1)   # top two well separated
        assert clear.any() and torch.equal(a.argmax(-1)[clear], b.argmax(-1)[clear])


# ---- refusals --------------------------------------------------------------------------------------------------------
@gpu
def test_refusals_change_nothing():
    from kvquant_b200 import decode as kd
    from kvquant_b200.rope import LengthDependentRotary
    pc = TP._paged(4, 32, 8, 3, 160, n_pool=4, max_pages=3, seed=3)     # cap 480 tokens per slot
    pt = pc.pages
    k, v = G._tokens(pc._tmpl, 600, 1)
    pc.append_chunks([0], k[:100], v[:100], [100])                     # 1 page, 3 free
    pc.commit()

    def state():
        return (_snapshot(pc), [list(r) for r in pt.pages], list(pt._free), list(pt.lens_host), pt.table.clone(),
                pt.npages.clone(), pt.lens.clone(), list(pt.refs))

    def same(a, b):
        return _equal(a[0], b[0]) and a[1:4] == b[1:4] and all(torch.equal(x, y) for x, y in zip(a[4:7], b[4:7])) \
            and a[7] == b[7]
    s0 = state()
    with pytest.raises(ValueError):                 # duplicate slots
        pc.append_chunks([1, 1], k[:20], v[:20], [10, 10])
    with pytest.raises(IndexError):                 # slot 1 past the cap
        pc.append_chunks([0, 1], k[:491], v[:491], [10, 481])
    with pytest.raises(RuntimeError):               # 2 + 2 pages wanted, 3 free
        pc.append_chunks([1, 2], k[:520], v[:520], [320, 200])
    assert same(s0, state())
    pc.append_chunks([1], k[:160], v[:160], [160])  # slot 1 fills one page ...
    pc.commit()
    pc.fork(1, 2)                                   # ... which slot 2 then shares
    s1 = state()
    with pytest.raises(RuntimeError):               # a write into the shared page
        pc._append_chunks_at([2, 0], [100, 100], k[:20], v[:20], [10, 10])
    assert same(s1, state())
    bc = TB._batch(4, 32, 8, 2, Lmax=160)
    bs = (_snapshot(bc), bc.lens_host, bc.lens.clone())
    with pytest.raises(IndexError):
        bc.append_chunks([0, 1], k[:400], v[:400], [100, 300])
    assert _equal(bs[0], _snapshot(bc)) and bc.lens_host == bs[1] and torch.equal(bc.lens, bs[2])
    # length-dependent rotary: refused by the cache and by the stage
    q = torch.zeros((10, 32, 128), device=DEV)
    spec = LengthDependentRotary(10000.0, {"rope_type": "dynamic", "factor": 2.0}, 4096)
    with pytest.raises(NotImplementedError):
        bc.attend_chunks([0], q, k[:10], v[:10], [10], rope=spec)
    _, quant = TB._stage("llama3_8b")
    cfg = kd.DecodeConfig.llama3_8b(n_layers=1, max_len=512, max_position_embeddings=4096,
                                    rope_scaling={"rope_type": "dynamic", "factor": 2.0})
    st = kd.DecoderStage(cfg, 0, 1, DEV, quant, seed=1, with_head=True)
    bst = kd.BatchedDecoderStage(st, 2)
    with pytest.raises(NotImplementedError):
        bst.prefill_seqs({0: st.embed[:5]})
    assert bst.lens.tolist() == [0, 0] and bst.caches[0].lens_host == [0, 0]
