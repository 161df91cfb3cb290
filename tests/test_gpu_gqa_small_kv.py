"""Two-KV-head and multi-query models over the quantised cache: H_kv in {1, 2} with H_q % 4 == 0, H_q <= 64.

Shapes (H_q, H_kv): (8, 1), (32, 1), (64, 1), (12, 2), (16, 2), (32, 2), (64, 2), and (32, 8) as a control.  The K
ratio kernel's sub-group CTAs (a KV head's query heads spread over several CTAs) run at 4 bits from 20 query heads per
KV head and at 3 / 2 bits from 36: (32, 1), (64, 1) and (64, 2) here.  The 3-bit V pass's padded box runs at H_kv = 1.

Most checks are the GQA, batch, paged, dequantisation and rotary tests of the other modules run at these shapes; what
only these shapes need (slots past the length, bit-exact appends at KV hidden 128 and 256, the decode harness at
n_kv_heads 1 and 2) is written out here.
"""
import numpy as np
import pytest
import torch

import test_gpu_append_edges as AE
import test_gpu_batch as TB
import test_gpu_dequant as DQ
import test_gpu_gqa as G
import test_gpu_paged as PG
import test_gpu_rope_length as RL
import test_gpu_rope_scaling as RS
from _util import quantizer, spec
from kvquant_b200 import synth

gpu = pytest.mark.gpu
DEV = G.DEV
SMALL = ((8, 1), (32, 1), (64, 1), (12, 2), (16, 2), (32, 2), (64, 2))
SHAPES = SMALL + ((32, 8),)
LENGTHS = (1, 31, 32, 33, 159, 160, 161, 4096, 20000)


# ---- decode attend against float64 -----------------------------------------------------------------------------------
@gpu
@pytest.mark.parametrize("mode", ["kv", "k", "dense"])
@pytest.mark.parametrize("Hq,Hkv", SHAPES)
@pytest.mark.parametrize("bits", [4, 3, 2])
def test_attend_against_float64(bits, Hq, Hkv, mode):
    lc = G._cache(bits, Hq, Hkv, mode, n_sink=5)
    lc.append_chunk(*G._tokens(lc, max(LENGTHS), seed=bits * 100 + Hq + Hkv))
    q = G._query(Hq, bits)
    for L in LENGTHS:
        lc.len = L
        for sinks in (False, True):
            lc.sink_k = lc.sink_v = None
            if sinks:
                G._sinks(lc, 5, seed=L)
            G._check(G._attend(lc, q), G._oracle_gqa(lc, q), "L=%d sinks=%s" % (L, sinks))


@gpu
@pytest.mark.parametrize("mode", ["kv", "dense"])
@pytest.mark.parametrize("Hq,Hkv", SMALL)
@pytest.mark.parametrize("bits", [4, 3, 2])
def test_attend_equals_replicated_mha(bits, Hq, Hkv, mode):
    G.test_attend_equals_replicated_mha(bits, Hq, Hkv, mode)


# ---- other decode forms -------------------------------------------------------------------------------------------------
@gpu
@pytest.mark.parametrize("Hq,Hkv", SMALL)
def test_attend_dyn_and_graph(Hq, Hkv):
    G.test_attend_dyn_matches_attend_and_graph_extends_the_cache(Hq, Hkv)


@gpu
@pytest.mark.parametrize("Hq,Hkv", SMALL)
def test_merge_of_two_halves(Hq, Hkv):
    G.test_merge_of_two_halves_equals_the_whole(Hq, Hkv)


@gpu
@pytest.mark.parametrize("mode", ("kv", "dense"))
@pytest.mark.parametrize("shape", ((64, 1), (32, 1), (16, 2), (64, 2)))
def test_batched_attend_agrees_with_attend_dyn(mode, shape):
    TB.test_batched_attend_agrees_with_attend_dyn_on_each_view(mode, shape)


@gpu
@pytest.mark.parametrize("shape", SMALL)
def test_batch_of_one_is_bit_identical_to_attend_dyn(shape):
    TB.test_batch_of_one_is_bit_identical_to_attend_dyn(shape)


@gpu
@pytest.mark.parametrize("B", (3, 8))
@pytest.mark.parametrize("bits,Hq,Hkv", ((4, 64, 1), (3, 64, 1), (3, 32, 2), (2, 64, 2)))
def test_batched_attend_per_sequence(bits, Hq, Hkv, B):
    lens = tuple((0, 1, 161, 4096, 777, 33, 20000, 160)[:B])
    bc = TB._batch(bits, Hq, Hkv, B, "kv")
    TB._fill(bc, lens, 70 + B)
    q = TB._queries(bc, 2)
    out, lse = TB._battend(bc, q, L_cap=G.LMAX)
    for b in range(B):
        if lens[b] == 0:
            continue
        o1, l1 = TB._view_attend(bc, b, q[b], G.LMAX)
        assert G._head_err(out[b].cpu().numpy(), o1.cpu().numpy()) < 4e-6, b
        assert float((lse[b] - l1).abs().max()) < 1e-6 * float(l1.abs().max() + 1), b


@gpu
@pytest.mark.parametrize("P", (160, 640))
@pytest.mark.parametrize("mode", ("kv", "dense"))
@pytest.mark.parametrize("case", ((4, 64, 1), (3, 32, 1), (3, 64, 2), (2, 16, 2), (4, 12, 2)))
def test_paged_attend_equals_the_contiguous_batch(case, mode, P):
    bits, Hq, Hkv = case
    lens = (1, 0, 333, 4096, 12345, 700)
    bc, pc, Lmax = PG._pair(bits, Hq, Hkv, lens, P, mode)
    q = TB._queries(pc, 2)
    out, lse = PG._pattend(pc, q, L_cap=Lmax)
    o1, l1 = TB._battend(bc, q, L_cap=Lmax)
    if mode == "dense":
        assert torch.equal(out, o1) and torch.equal(lse, l1)
    else:
        assert TB._close(out, o1)
        live = torch.isfinite(l1)
        assert torch.equal(torch.isfinite(lse), live)
        assert float((lse - l1)[live].abs().max()) < 1e-6 * float(l1[live].abs().max() + 1)
    assert torch.equal(out[1], torch.zeros_like(out[1])) and bool(torch.isneginf(lse[1]).all())


# ---- exact probes -------------------------------------------------------------------------------------------------------
@gpu
@pytest.mark.parametrize("Hq,Hkv", ((16, 2), (64, 2), (32, 2)))
def test_poisoned_kv_head_reaches_only_its_query_heads(Hq, Hkv):
    G.test_poisoned_kv_head_reaches_only_its_query_heads(Hq, Hkv)


@gpu
@pytest.mark.parametrize("mode", ("dense", "kv"))
@pytest.mark.parametrize("Hq,Hkv", SMALL)
@pytest.mark.parametrize("bits", [4, 3])
def test_slots_past_the_length_are_never_read(bits, Hq, Hkv, mode):
    """Huge words, NaN outlier rows and NaN (sf, off) in every slot past the length change nothing: bit for bit on a
    dense cache, within 1e-6 of each head's max where the V outlier reductions may land in another order."""
    lc = G._cache(bits, Hq, Hkv, mode, Lmax=4096, n_sink=3)
    G._sinks(lc, 3, seed=1)
    lc.append_chunk(*G._tokens(lc, 3000, seed=5))
    q = G._query(Hq, 3)
    for L in (1, 161, 2911):
        lc.len = L
        base, lbase = (x.clone() for x in G._attend(lc, q))
        dyn = G._attend(lc, q, dyn=L)[0].clone()
        saved = {n: getattr(lc, n).clone() for n in PG._tensors(lc)}
        gen = torch.Generator(device=DEV).manual_seed(L)
        for n in ("kcache", "vcache"):
            t = getattr(lc, n)[..., L:]
            t.copy_(torch.randint(-2 ** 31, 2 ** 31 - 1, t.shape, generator=gen, device=DEV, dtype=torch.int32))
        lc.vaff[L:] = float("nan")
        for side in ("k", "v"):
            if getattr(lc, "sparse_" + side):
                getattr(lc, side + "_outliers")[L:] = float("nan")
        got, lgot = G._attend(lc, q)
        got_dyn = G._attend(lc, q, dyn=L)[0]
        if mode == "dense":
            assert torch.equal(got, base) and torch.equal(lgot, lbase) and torch.equal(got_dyn, dyn), L
        else:
            assert torch.isfinite(got).all() and torch.isfinite(got_dyn).all(), L
            assert G._head_err(got.cpu().numpy(), base.cpu().numpy()) <= 1e-6, L
            assert G._head_err(got_dyn.cpu().numpy(), dyn.cpu().numpy()) <= 1e-6, L
        for n, t in saved.items():
            getattr(lc, n).copy_(t)


# ---- appends at KV hidden 128 and 256 -------------------------------------------------------------------------------------
@gpu
@pytest.mark.parametrize("H", (1, 2))
@pytest.mark.parametrize("bits", (2, 3, 4))
def test_append_bit_exact_against_the_oracle(bits, H):
    """Codes, outlier rows and V (sf, off) against the strict-rule numpy oracle (the outlier budget of hidden 128 / 256
    at t = 0.99: n_each = 1 / 2), the last 20 tokens through the device-length append; append_chunk of the same tokens
    in two chunks equals the single appends bit for bit."""
    from kvquant_b200.cache import LayerCache
    L = 200
    k, v = spec(H).k_tokens(L, seed=31), spec(H).v_tokens(L, seed=32)
    c, lc = AE.fill(bits, H, 256, k, v, n_dyn=20)
    assert lc.n_out == 2 * H
    AE.assert_state_matches(lc, c)
    klut, vcent = quantizer(bits, H=H)
    ch = LayerCache.from_luts(bits, H, 256, klut, vcent, device=DEV)
    ch.append_chunk(AE.cu(k[:150]), AE.cu(v[:150]))
    ch.append_chunk(AE.cu(k[150:]), AE.cu(v[150:]))
    assert ch.len == L
    for name in PG._tensors(lc):
        assert torch.equal(getattr(ch, name), getattr(lc, name)), name


@gpu
@pytest.mark.parametrize("B", (1, 8))
@pytest.mark.parametrize("mode", ("kv", "k", "dense"))
@pytest.mark.parametrize("shape", ((8, 1), (64, 2)))
@pytest.mark.parametrize("bits", (2, 3, 4))
def test_batched_append_is_bit_identical_to_single_appends(bits, shape, mode, B):
    TB.test_batched_append_is_bit_identical_to_single_appends(bits, mode, shape, B)


@gpu
@pytest.mark.parametrize("mode", ("kv", "dense"))
@pytest.mark.parametrize("shape", ((32, 1), (16, 2)))
@pytest.mark.parametrize("bits", (2, 3, 4))
def test_paged_append_is_bit_identical_to_the_contiguous_batch(bits, shape, mode):
    PG.test_paged_append_is_bit_identical_to_the_contiguous_batch(bits, mode, shape)


# ---- readers of the cache -----------------------------------------------------------------------------------------------
@gpu
@pytest.mark.parametrize("H", (1, 2))
@pytest.mark.parametrize("bits,mode", ((4, "kv"), (3, "kv"), (2, "kv"), (4, "dense"), (4, "k_only")))
def test_dequantize_against_the_oracle(bits, mode, H):
    DQ.test_prerope_k_bit_exact_and_v_within_one_ulp(bits, H, mode, False)


@gpu
@pytest.mark.parametrize("H", (1, 2))
@pytest.mark.parametrize("bits", (4, 3, 2))
def test_rotated_dequantize_against_float64(bits, H):
    DQ.test_rotated_k_against_float64_rotation(bits, H, 5, 77, 10000.0)


@gpu
@pytest.mark.parametrize("Hq,Hkv", ((32, 1), (16, 2)))
@pytest.mark.parametrize("bits", (4, 3))
def test_paged_dequantize_equals_contiguous(bits, Hq, Hkv):
    lens = (333, 1000)
    bc, pc, _ = PG._pair(bits, Hq, Hkv, lens, 160, "kv")
    for b, n in enumerate(lens):
        for theta in (None, 10000.0):
            want = bc.seq(b).dequantize(0, n, rope_theta=theta)
            got = pc.dequantize(b, 0, n, rope_theta=theta)
            assert torch.equal(got[0], want[0]) and torch.equal(got[1], want[1]), (b, theta)


@gpu
@pytest.mark.parametrize("mode", ["kv", "dense"])
@pytest.mark.parametrize("Hq,Hkv", SMALL)
@pytest.mark.parametrize("bits", [4, 3, 2])
def test_chunk_attends_against_float64(bits, Hq, Hkv, mode):
    G.test_chunk_attends_against_float64(bits, Hq, Hkv, mode)


@gpu
@pytest.mark.parametrize("bits", [4, 3])
def test_scaled_rotary(bits):
    RS.test_attend_against_float64(bits, 16, 2, "kv", sorted(RS.SPECS)[0])


@gpu
@pytest.mark.parametrize("bits", [4, 3])
def test_length_dependent_rotary(bits):
    RL.test_attend_against_float64(bits, 16, 2, "kv")


# ---- decode harness -----------------------------------------------------------------------------------------------------
def _quant(kv_heads):
    from kvquant_b200 import cache as kc
    sp = synth.SynthSpec(kv_heads, 128, seed=0)
    cal = synth.calibrate(sp, 4, calib_tokens=256, seed=7)
    t = kc.build_k_lookup_table(cal["k"][0], cal["k"][1], cal["k"][2][0], kv_heads, device=DEV)
    return dict(klut=dict(lut=t["lut"], lut2=None, thr_lower=t["thr_lower"], thr_upper=t["thr_upper"]),
                v_cent=cal["v"][2][0])


@gpu
def test_two_kv_head_stage_prefills_then_decodes_in_one_graph():
    from kvquant_b200 import decode as kd
    cfg = kd.DecodeConfig(n_layers=2, hidden=2048, n_heads=16, n_kv_heads=2, intermediate=5632, vocab=32000,
                          rope_theta=1e6, max_len=4096, n_sink=2)
    st = kd.DecoderStage(cfg, 0, 2, DEV, _quant(2), seed=1, with_head=True)
    assert st.layers[0].wqkv.shape == (20 * 128, 2048) and st.layers[0].cache.sink_k.shape == (2, 128, 2)
    toks = torch.randint(0, cfg.vocab, (1000,), generator=torch.Generator().manual_seed(0)).to(DEV)
    st.prefill(st.embed[toks], chunk=384)
    L = st.layers[0].cache.len
    assert L == 1000
    gs = kd.GraphedStage(st, L, first=True, last_to_logits=True, dynamic=True)
    steps = [int(x) for x in torch.randint(0, cfg.vocab, (16,), generator=torch.Generator().manual_seed(1))]
    got = []
    for tok in steps:
        gs.tok.fill_(tok)
        gs.replay()
        torch.cuda.synchronize()
        got.append(gs.logits.clone())
    assert st.layers[0].cache.len == L + 16
    st.dyn = None
    st.set_len(L)
    for i, tok in enumerate(steps):
        ref = st.head(st.forward_torch(st.embed_token(torch.tensor([tok], device=DEV))))
        assert torch.isfinite(got[i].float()).all()
        d = (ref.float() - got[i].float()).abs().max().item()
        assert d <= 1e-2 * max(1.0, ref.float().abs().max().item()), (i, d)


@gpu
def test_multi_query_paged_batched_stage_prefills_forks_and_steps():
    from kvquant_b200 import decode as kd
    cfg = kd.DecodeConfig(n_layers=2, hidden=2048, n_heads=16, n_kv_heads=1, intermediate=5632, vocab=32000,
                          max_len=1280, n_sink=2)
    st = kd.DecoderStage(cfg, 0, 2, DEV, _quant(1), seed=1, with_head=True)
    bst = kd.BatchedDecoderStage(st, 4, page_size=160, n_pool=40)
    gen = torch.Generator().manual_seed(3)
    prompts = [torch.randint(0, cfg.vocab, (n,), generator=gen).to(DEV) for n in (300, 37, 161)]
    for b, p in enumerate(prompts):
        bst.prefill_seq(b, st.embed[p], chunk=128)
    bst.fork_seq(0, 3)
    assert bst.lens.tolist() == [300, 37, 161, 300]
    g = kd.BatchedGraphedStep(bst)
    toks = torch.randint(0, cfg.vocab, (6, 4), generator=gen)
    toks[:, 3] = toks[:, 0]              # the fork follows its source token for token
    got = []
    for i in range(6):
        g.tok.copy_(toks[i].to(DEV))
        g.replay()
        torch.cuda.synchronize()
        got.append(g.logits.float().clone())
    assert bst.lens.tolist() == [306, 43, 167, 306]
    for i in range(6):
        assert torch.isfinite(got[i]).all(), i
        assert torch.equal(got[i][0], got[i][3]), i
    ref = TB._single_reference(st, prompts[1], toks[:, 1].tolist())
    for i in range(6):
        d = (ref[i] - got[i][1]).abs().max().item()
        assert d <= 1e-2 * max(1.0, ref[i].abs().max().item()), (i, d)
