"""GPU: attends over the quantised cache with length-dependent rotary frequencies (dynamic NTK, LongRoPE; DESIGN.md
section 4.14).  Every key and the query are rotated with f(s), s = one plus the position of the call's last query.

* the rotation state: after kvq_rope_len_update at s, the table equals kvq_rope_table_build_freq over the host f(s)
  bit for bit (below M, at M, M + 1, far past M, and back below), and f_cur equals the host f(s) across M;
* attend / attend_dyn equal the *_freq attends over a static table built from f(s): bit for bit on dense caches,
  within the few-ulp agreement of section 4.10 with outliers; the batched and paged attends with slots on both sides
  of M equal single-sequence attends;
* attends against a float64 oracle whose cos / sin come from the host f(s), at tests/test_gpu_gqa.py's tolerances;
  dequantize against float64 rotate-half at f(len), the chunk attends against float64 causal attention at f(len + T);
* a result straddling M differs from the static theta result (the old keys were rotated again);
* a one-graph dynamic decode crossing M follows the eager step; a paged BatchedGraphedStep at B = 3 with slots below,
  at and above M follows single-sequence runs through reset_seq, prefill_seq and fork_seq;
* sinks, fp16 tables, sequence-sharded and layer-pipelined stages are refused.
"""
import numpy as np
import pytest
import torch

import test_gpu_gqa as G
from kvquant_b200 import _lib, quant_cuda as qc
from kvquant_b200.cache import RopeLenState
from kvquant_b200.rope import LengthDependentRotary

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
M = 4096
DYN = LengthDependentRotary(10000.0, {"rope_type": "dynamic", "factor": 2.0}, M)
LONG = LengthDependentRotary(10000.0, {"rope_type": "longrope", "original_max_position_embeddings": M,
                                       "long_factor": [1.0 + 0.03125 * i for i in range(64)],
                                       "short_factor": [1.0 + 0.0078125 * (i % 7) for i in range(64)]}, 4 * M)
SPECS = {"dynamic": DYN, "longrope": LONG}


def static_table(spec, s, npos):
    f = spec.inv_freq_at(s).to(DEV)
    t = torch.empty((64, npos, 2), dtype=torch.float32, device=DEV)
    _lib.check(_lib.load().kvq_rope_table_build_freq(t.data_ptr(), f.data_ptr(), float(spec.attention_factor), npos,
                                                     torch.cuda.current_stream().cuda_stream), "build_freq")
    return t, f


def cos_sin64(spec, s, p0, L):
    """float64 cos / sin of the fp32 angle f(s)_j * p, times the attention factor: [128, L] each."""
    f = spec.inv_freq_at(s).numpy()
    p = np.arange(p0, p0 + L, dtype=np.float32)
    ang = (f[:, None] * p[None, :]).astype(np.float32).astype(np.float64)
    a = spec.attention_factor
    c, sn = np.cos(ang) * a, np.sin(ang) * a
    return np.concatenate([c, c]), np.concatenate([sn, sn])


def rotate_q(spec, s, q, pos):
    c, sn = cos_sin64(spec, s, pos, 1)
    q = q.double().cpu().numpy()
    rot = np.concatenate([-q[:, 64:], q[:, :64]], axis=1)
    return torch.from_numpy((q * c[:, 0] + rot * sn[:, 0]).astype(np.float32)).to(DEV)


def oracle(lc, q, spec, s):
    st = G._state(lc)
    st["cos_sin"] = cos_sin64(spec, s, lc.n_sink + lc.pos_base, lc.len)
    return G._oracle_gqa(lc, q, st)


# ---- the rotation state -------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name", sorted(SPECS))
def test_state_table_equals_the_static_build_at_every_step(name):
    spec = SPECS[name]
    npos = 3 * M
    st = RopeLenState(spec, 1, npos, DEV)
    for s in (100, M - 1, M, M + 1, M + 2, 3 * M - 7, M + 1, 50, M):
        st.update(s=s)
        torch.cuda.synchronize()
        want, f = static_table(spec, s, st.npos)
        assert torch.equal(st.f_cur[0], f), (name, s)
        assert torch.equal(st.table[0][:, :s], want[:, :s]), (name, s)
    for s in range(M - 40, M + 40):
        st.update(s=s)
        assert torch.equal(st.f_cur[0].cpu(), spec.inv_freq_at(s)), (name, s)


def test_device_f_equals_host_f_far_past_the_switch():
    st = RopeLenState(DYN, 1, 1 << 20, DEV)
    for s in list(range(M + 1, M + 400)) + [2 ** k for k in range(13, 21)]:
        st.update(s=s)
        assert torch.equal(st.f_cur[0].cpu(), DYN.inv_freq_at(s)), s


def test_batched_state_reads_each_sequence_length():
    st = RopeLenState(DYN, 3, 2 * M, DEV)
    lens = torch.tensor([M - 3, M - 1, M + 5], dtype=torch.int64, device=DEV)
    st.update(len_dev=lens, len_add=1, L_cap=2 * M - 1, pos_offset=0)
    torch.cuda.synchronize()
    for b, L in enumerate(lens.tolist()):
        want, f = static_table(DYN, L + 1, st.npos)
        assert torch.equal(st.f_cur[b], f) and torch.equal(st.table[b][:, :L + 1], want[:, :L + 1]), b


# ---- attends against the static *_freq attend ----------------------------------------------------------------------
@pytest.mark.parametrize("name", sorted(SPECS))
@pytest.mark.parametrize("mode", ["dense", "kv"])
def test_attend_equals_the_static_freq_attend(name, mode):
    spec = SPECS[name]
    lc = G._cache(3, 32, 8, mode, Lmax=M + 104, n_sink=0)
    lc.append_chunk(*G._tokens(lc, M + 100, seed=4))
    for L in (M - 2, M - 1, M, M + 1, M + 100):
        lc.len = L
        q = G._query(32, L)
        got = lc.attend(q, rope=spec).clone()
        dyn = lc.attend_dyn(q, torch.full((1,), L - 1, dtype=torch.int64, device=DEV), 1, L_cap=M + 104,
                            rope=spec).clone()
        t, f = static_table(spec, L, L + 1)
        # the same attend over the static table and vector (the *_freq entry point)
        from kvquant_b200 import cache as kc
        orig = kc._rope_call
        kc._rope_call = lambda dev, r: ("_freq", (f.data_ptr(), float(spec.attention_factor)))
        qc_tables = qc.rope_tables
        qc.rope_tables = lambda dev, th, n: (t, None, t.shape[1])
        try:
            want = lc._attend(q, None, 0, 1.0, None, None, L).clone()
        finally:
            kc._rope_call, qc.rope_tables = orig, qc_tables
        if mode == "dense":
            assert torch.equal(got, want) and torch.equal(dyn, want), (name, L)
        else:
            assert (got - want).abs().max().item() <= 1e-5 * want.abs().max().item(), (name, L)
            assert (dyn - want).abs().max().item() <= 1e-5 * want.abs().max().item(), (name, L)


# ---- attends against float64 ---------------------------------------------------------------------------------------
LENGTHS = (33, M - 1, M, M + 1, M + 900)


@pytest.mark.parametrize("mode", ["kv", "k", "dense"])
@pytest.mark.parametrize("Hq,Hkv", [(32, 32), (32, 8)])
@pytest.mark.parametrize("bits", [4, 3, 2])
def test_attend_against_float64(bits, Hq, Hkv, mode):
    for name, spec in sorted(SPECS.items()):
        lc = G._cache(bits, Hq, Hkv, mode, Lmax=M + 904, n_sink=0)
        lc.append_chunk(*G._tokens(lc, max(LENGTHS), seed=bits * 100 + Hq))
        for L in LENGTHS:
            lc.len = L
            q = rotate_q(spec, L, G._query(Hq, L), L - 1)
            out, lse = torch.empty((Hq, 128), device=DEV), torch.empty(Hq, device=DEV)
            lc.attend(q, out=out, lse=lse, rope=spec)
            want = oracle(lc, q, spec, L)
            G._check((out, lse), want, "%s L=%d" % (name, L))
            out2, lse2 = torch.empty_like(out), torch.empty_like(lse)
            lc.attend_dyn(q, torch.full((1,), L - 3, dtype=torch.int64, device=DEV), 3, out=out2, lse=lse2,
                          L_cap=M + 900, rope=spec)
            G._check((out2, lse2), want, "%s dyn L=%d" % (name, L))
        # a result straddling the switch differs from the static theta rotation: the old keys were rotated again
        if name == "dynamic":
            plain = lc.attend(q, rope_theta=10000.0).cpu().numpy()
            assert G._head_err(plain, want[0]) > 100 * G.EXACT_TOL


@pytest.mark.parametrize("paged", [False, True])
@pytest.mark.parametrize("name", sorted(SPECS))
def test_batched_attends_against_float64(name, paged):
    from kvquant_b200 import cache as kc
    spec = SPECS[name]
    bits, Hq, Hkv, B, Lmax = 3, 32, 8, 3, M + 320
    tmpl = G._cache(bits, Hq, Hkv, "kv", Lmax=Lmax, n_sink=0)
    lens = (M - 40, M - 1, M + 200)                 # s = L: below, at and above the switch
    if paged:
        pt = kc.PageTable(B, 160, B * Lmax // 160, Lmax // 160, DEV)
        bc = kc.PagedLayerCache(B, bits, Hkv, tmpl.klut, None, tmpl.thr_lower, tmpl.thr_upper, tmpl.v_cent, DEV, True,
                                0.99, 0, None, True, Hq, pages=pt)
    else:
        bc = kc.BatchedLayerCache(B, bits, Hkv, Lmax, tmpl.klut, None, tmpl.thr_lower, tmpl.thr_upper, tmpl.v_cent,
                                  DEV, True, 0.99, 0, None, True, Hq)
    qs = []
    for b, L in enumerate(lens):
        k, v = G._tokens(tmpl, L, seed=b)
        if paged:
            bc.append_chunk(b, k, v)
        else:
            bc.seq(b).append_chunk(k, v)
        bc.commit(b)
        qs.append(rotate_q(spec, L + 1, G._query(Hq, b), L))
    out, lse = torch.empty((B, Hq, 128), device=DEV), torch.empty((B, Hq), device=DEV)
    # len_add = 1: each sequence attends one slot past its length, as a decode step after its append
    for b, L in enumerate(lens):
        k1, v1 = G._tokens(tmpl, 1, seed=50 + b)
        if paged:
            bc.pages.reserve(b, L + 1)
            bc.append_chunk(b, k1, v1)
            bc.pages.lens_host[b] = L
        else:
            bc.seq(b).append_chunk(k1, v1)
            bc.seq(b).len = L
        bc.commit(b)
    wants = []
    for b, L in enumerate(lens):
        ref = G._cache(bits, Hq, Hkv, "kv", Lmax=Lmax, n_sink=0)
        k, v = G._tokens(tmpl, L, seed=b)
        k1, v1 = G._tokens(tmpl, 1, seed=50 + b)
        ref.append_chunk(torch.cat([k, k1]), torch.cat([v, v1]))
        wants.append(oracle(ref, qs[b], spec, L + 1))
    bc.attend(torch.stack(qs), out=out, lse=lse, len_add=1, rope=spec)
    torch.cuda.synchronize()
    for b in range(B):
        G._check((out[b], lse[b]), wants[b], "b=%d" % b)
        single = G._cache(bits, Hq, Hkv, "kv", Lmax=Lmax, n_sink=0)
        k, v = G._tokens(tmpl, lens[b], seed=b)
        k1, v1 = G._tokens(tmpl, 1, seed=50 + b)
        single.append_chunk(torch.cat([k, k1]), torch.cat([v, v1]))
        one = single.attend(qs[b], rope=spec)
        assert (one - out[b]).abs().max().item() <= 1e-5 * one.abs().max().item(), b


@pytest.mark.parametrize("name", sorted(SPECS))
def test_dequantize_and_chunk_attends(name):
    spec = SPECS[name]
    L0 = M - 30
    lc = G._cache(4, 32, 8, "kv", Lmax=M + 104, n_sink=0)
    lc.append_chunk(*G._tokens(lc, L0, seed=1))
    pre, _ = lc.dequantize(0, L0)
    rot, _ = lc.dequantize(0, L0, rope=spec)
    c, s = cos_sin64(spec, L0, 0, L0)
    k = pre.double().cpu().numpy()
    kr = np.concatenate([-k[..., 64:], k[..., :64]], axis=-1)
    want = k * c.T[None] + kr * s.T[None]
    assert np.abs(rot.double().cpu().numpy() - want).max() <= 2.0 ** -9 * np.abs(want).max()
    T = 96                                                        # L0 + T straddles M: f(len + T) is past the switch
    kc_, vc_ = G._tokens(lc, T, seed=2)
    S_end = L0 + T
    q = torch.stack([rotate_q(spec, S_end, G._query(32, i), L0 + i) for i in range(T)])
    a = lc.attend_chunk(q, kc_, vc_, rope=spec)
    b = lc.attend_chunk_fused(q, kc_, vc_, rope=spec)
    cc, ss = cos_sin64(spec, S_end, 0, S_end)
    kall = np.concatenate([pre.double().cpu().numpy(),
                           kc_.view(T, 8, 128).double().cpu().numpy().transpose(1, 0, 2)], 1)   # [8, S, 128]
    kallr = np.concatenate([-kall[..., 64:], kall[..., :64]], axis=-1)
    K = kall * cc.T[None] + kallr * ss.T[None]
    K = K.astype(np.float16).astype(np.float64)          # both chunk attends read fp16 rotated keys
    _, vpre = lc.dequantize(0, L0)
    V = np.concatenate([vpre.double().cpu().numpy(),
                        vc_.view(T, 8, 128).half().double().cpu().numpy().transpose(1, 0, 2)], 1)
    qn = q.half().double().cpu().numpy()
    Sc = np.einsum("thc,hsc->ths", qn, np.repeat(K, 4, axis=0)) / np.sqrt(128.0)
    mask = np.arange(S_end)[None, :] <= (L0 + np.arange(T))[:, None]
    Sc = np.where(mask[:, None, :], Sc, -np.inf)
    P = np.exp(Sc - Sc.max(-1, keepdims=True))
    O = np.einsum("ths,hsc->thc", P, np.repeat(V, 4, axis=0)) / P.sum(-1)[..., None]
    scale = np.abs(O).max()
    for got in (a, b):
        assert np.abs(got.double().cpu().numpy() - O).max() <= 2e-3 * scale


# ---- refusals -----------------------------------------------------------------------------------------------------
def test_refusals():
    lc = G._cache(3, 32, 8, "kv", Lmax=1024, n_sink=2)
    lc.append_chunk(*G._tokens(lc, 100, seed=1))
    with pytest.raises(NotImplementedError, match="sinks"):
        lc.attend(G._query(32, 1), rope=DYN)
    lc2 = G._cache(3, 32, 32, "kv", Lmax=1024, n_sink=0)
    lc2.append_chunk(*G._tokens(lc2, 100, seed=1))
    lc2.precision = "fp16"
    with pytest.raises(NotImplementedError, match="fp32"):
        lc2.attend(G._query(32, 1), rope=DYN)
    from kvquant_b200 import decode as kd
    cfg = kd.DecodeConfig.llama3_8b(n_layers=1, max_len=256, rope_scaling={"rope_type": "dynamic", "factor": 2.0},
                                    max_position_embeddings=128)
    with pytest.raises(NotImplementedError):
        kd.DecoderStage(cfg, 0, 1, DEV, _quant(), sp=(0, 2))
    st = kd.DecoderStage(cfg, 0, 1, DEV, _quant())
    with pytest.raises(NotImplementedError):
        kd.GraphedStage(st, 0, True, True, pp=(0, 2))


# ---- the decode harness --------------------------------------------------------------------------------------------
def _quant():
    from kvquant_b200 import cache as kc, synth
    sp = synth.SynthSpec(8, 128, seed=0)
    cal = synth.calibrate(sp, 4, calib_tokens=256, seed=7)
    t = kc.build_k_lookup_table(cal["k"][0], cal["k"][1], cal["k"][2][0], 8, device=DEV)
    return dict(klut=dict(lut=t["lut"], lut2=None, thr_lower=t["thr_lower"], thr_upper=t["thr_upper"]),
                v_cent=cal["v"][2][0])


def _stage(Mpe, n_layers=2, max_len=1280):
    from kvquant_b200 import decode as kd
    cfg = kd.DecodeConfig.llama3_8b(n_layers=n_layers, max_len=max_len, n_sink=0,
                                    rope_scaling={"rope_type": "dynamic", "factor": 4.0}, max_position_embeddings=Mpe)
    return kd.DecoderStage(cfg, 0, n_layers, DEV, _quant(), seed=1, with_head=True)


def _close(ref, got, what):
    ref, got = ref.float(), got.float()
    d = (ref - got).abs().max().item()
    assert torch.isfinite(got).all() and d <= 1e-2 * max(1.0, ref.abs().max().item()), (what, d)


def test_one_graph_dynamic_decode_crosses_the_switch():
    from kvquant_b200 import decode as kd
    Mpe = 1000
    st = _stage(Mpe)
    toks = torch.randint(0, st.cfg.vocab, (Mpe - 4,), generator=torch.Generator().manual_seed(0)).to(DEV)
    st.prefill(st.embed[toks], chunk=4096)
    L = st.layers[0].cache.len                      # the first step's s = L + 1 = M - 3
    gs = kd.GraphedStage(st, L, first=True, last_to_logits=True, dynamic=True)
    steps = [int(x) for x in torch.randint(0, st.cfg.vocab, (9,), generator=torch.Generator().manual_seed(1))]
    got = []
    for tok in steps:
        gs.tok.fill_(tok)
        gs.replay()
        torch.cuda.synchronize()
        got.append(gs.logits.clone())
    st.dyn = None
    st.set_len(L)
    for i, tok in enumerate(steps):
        eager = st.head(st.forward(st.embed_token(torch.tensor([tok], device=DEV))))
        _close(eager, got[i], "eager step %d" % i)
    st.set_len(L)
    for i, tok in enumerate(steps):
        ref = st.head(st.forward_torch(st.embed_token(torch.tensor([tok], device=DEV))))
        _close(ref, got[i], "torch step %d" % i)


def test_paged_batched_graph_follows_single_sequences_across_the_switch():
    from kvquant_b200 import decode as kd
    Mpe = 600
    st = _stage(Mpe, max_len=960)
    gen = torch.Generator().manual_seed(2)
    prompts = [torch.randint(0, st.cfg.vocab, (n,), generator=gen).to(DEV) for n in (Mpe - 8, Mpe - 1, Mpe + 20)]
    p3, suffix = (torch.randint(0, st.cfg.vocab, (n,), generator=gen).to(DEV) for n in (Mpe + 5, 7))
    A = torch.randint(0, st.cfg.vocab, (3, 3), generator=gen)
    Bt = torch.randint(0, st.cfg.vocab, (3, 3), generator=gen)
    bst = kd.BatchedDecoderStage(st, 3, page_size=160)
    for b, p in enumerate(prompts):
        bst.prefill_seq(b, st.embed[p], chunk=4096)
    g = kd.BatchedGraphedStep(bst)
    got = []

    def run(toks):
        for i in range(toks.shape[0]):
            g.tok.copy_(toks[i].to(DEV))
            g.replay()
            torch.cuda.synchronize()
            got.append(g.logits.float().clone())
    run(A)
    bst.reset_seq(0)
    bst.prefill_seq(0, st.embed[p3], chunk=4096)
    bst.reset_seq(1)
    bst.fork_seq(2, 1)
    bst.prefill_seq(1, st.embed[suffix], chunk=4096)
    run(Bt)
    # single-sequence histories: (prompt chunks and decode tokens), and the replays whose logits they must give
    hist = {0: [("p", prompts[0]), ("d", A[:, 0], 0)],
            1: [("p", prompts[1]), ("d", A[:, 1], 0)],
            2: [("p", prompts[2]), ("d", A[:, 2], 0), ("d", Bt[:, 2], 3)]}
    hist_b = {0: [("p", p3), ("d", Bt[:, 0], 3)],
              1: [("p", prompts[2]), ("x", A[:, 2]), ("p", suffix), ("d", Bt[:, 1], 3)]}
    for b, h in list(hist.items()) + [(("b", k), v) for k, v in hist_b.items()]:
        slot = b if isinstance(b, int) else b[1]
        st.set_len(0)
        for step in h:
            if step[0] == "p":
                st.prefill(st.embed[step[1]], chunk=4096)
            else:
                for i, tok in enumerate(step[1].tolist()):
                    ref = st.head(st.forward_torch(st.embed_token(torch.tensor([tok], device=DEV))))
                    if step[0] == "d" and not (isinstance(b, int) and b != 2 and step[2] == 3):
                        _close(ref, got[step[2] + i][slot], "slot %s step %d" % (b, step[2] + i))
