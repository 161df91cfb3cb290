"""GPU: attends over the quantised cache with scaled rotary frequencies (LLaMA-3.1 llama3, linear, YaRN).

* the freq-built f32 table equals float64 cos / sin(f_j p) * a (fp32 argument f_j p, as HF forms it) for all 64 rows;
* the outlier pass's computed factors equal the table's gather, bit for bit: attend outputs with every factor computed
  past CUDART_TRIG_PLOSS_F's row limits against the same attends with every factor gathered (KVQ_KOUT_DIRECT_NPOS in a
  subprocess), at positions straddling 105615 / f_j;
* attend, attend_dyn, BatchedLayerCache.attend and PagedLayerCache.attend against a float64 oracle whose cos / sin
  come from HF's fp32 f (not from the library's table), at the tolerances of tests/test_gpu_gqa.py, across 4/3/2 bits,
  MHA 32/32 and GQA 32/8, dense / K / K+V outliers, with and without sinks, lengths spanning 8192 and a 4K cache placed
  near position 128K;
* dequantize(rope=spec) against HF's apply_rotary_pos_emb in float64, attend_chunk / attend_chunk_fused against
  float64 causal attention;
* scaled and unscaled results differ at long positions; RotarySpec(theta) is bit-identical to rope_theta=theta;
* a llama31_8b-shaped stage: the one-graph dynamic decode after prefill follows the eager step, a paged
  BatchedGraphedStep at B = 2 follows single-sequence runs, prefill_seq into a forked slot.
"""
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

import test_gpu_gqa as G
from kvquant_b200.rope import RotarySpec

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
HERE = os.path.dirname(os.path.abspath(__file__))
LLAMA31 = RotarySpec(500000.0, {"rope_type": "llama3", "factor": 8.0, "low_freq_factor": 1.0, "high_freq_factor": 4.0,
                                "original_max_position_embeddings": 8192})
LINEAR8 = RotarySpec(10000.0, {"rope_type": "linear", "factor": 8.0})
YARN4 = RotarySpec(1000000.0, {"rope_type": "yarn", "factor": 4.0, "original_max_position_embeddings": 32768})
SPECS = {"llama3": LLAMA31, "linear": LINEAR8, "yarn": YARN4}
TRIG_FAST_MAX = 105615.0


def cos_sin64(spec, p0, L):
    """float64 cos / sin of HF's fp32 angle f_j * p, times the attention factor: [128, L] each (rotate-half rows)."""
    f = spec.inv_freq.numpy()
    p = np.arange(p0, p0 + L, dtype=np.float32)
    ang = (f[:, None] * p[None, :]).astype(np.float32).astype(np.float64)
    a = spec.attention_factor
    c, s = np.cos(ang) * a, np.sin(ang) * a
    return np.concatenate([c, c]), np.concatenate([s, s])


def rotate_q(spec, q, pos):
    """HF apply_rotary_pos_emb on the query in float64 (from the fp32 angle), rounded to fp32."""
    c, s = cos_sin64(spec, pos, 1)
    q = q.double().cpu().numpy()
    rot = np.concatenate([-q[:, 64:], q[:, :64]], axis=1)
    return torch.from_numpy((q * c[:, 0] + rot * s[:, 0]).astype(np.float32)).to(DEV)


def oracle(lc, q, spec):
    st = G._state(lc)
    st["cos_sin"] = cos_sin64(spec, lc.n_sink + lc.pos_base, lc.len)
    return G._oracle_gqa(lc, q, st)


# ---- tables -----------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name", sorted(SPECS))
def test_freq_table_against_float64(name):
    from kvquant_b200 import quant_cuda as qc
    spec = SPECS[name]
    n = (1 << 20) + 1
    t, th, npos = qc.rope_tables(torch.device(DEV), spec, n)
    for p0 in range(0, n, 1 << 18):
        L = min(1 << 18, n - p0)
        c, s = cos_sin64(spec, p0, L)
        got = t[:, p0:p0 + L].double().cpu().numpy()
        # fp32 cosf / sinf of the same fp32 argument: a couple of ulps, times a
        tol = 4 * 2.0 ** -24 * spec.attention_factor
        assert np.abs(got[..., 0] - c[:64]).max() <= tol and np.abs(got[..., 1] - s[:64]).max() <= tol, (name, p0)
    half = th[:, :4096].contiguous().view(torch.float16).view(64, 4096, 2).float()
    assert torch.equal(half, t[:, :4096].half().float())


# ---- outlier factors: computed == gathered ------------------------------------------------------------------------------
def _row_limit(spec, j):
    return int(TRIG_FAST_MAX / float(spec.inv_freq[j])) + 1


def _kout_case(name, j):
    """attend output of a 4K K-outlier cache (MHA 32 heads, 2 bits) placed so that its positions straddle row j's
    fast-reduction limit.  (K outliers only: the V outlier pass adds many tokens into one output with atomics, in no
    fixed order; the K pass adds at most two partial sums per score, which commute.)"""
    spec = SPECS[name]
    lc = G._cache(2, 32, 32, "k", Lmax=4096)
    lc.append_chunk(*G._tokens(lc, 4096, seed=j))
    lc.pos_base = max(0, _row_limit(spec, j) - 2048)
    q = rotate_q(spec, G._query(32, j), lc.pos_base + 4096)
    out = torch.empty((32, 128), device=DEV)
    lc.attend(q, out=out, rope=spec)
    torch.cuda.synchronize()
    return out.cpu().numpy()


KOUT = [(name, j) for name in sorted(SPECS) for j in (0, 1, 15) if _row_limit(SPECS[name], j) < (1 << 20)]
CHILD = r"""
import sys
sys.path.insert(0, %r)
import numpy as np
import test_gpu_rope_scaling as T
np.savez(sys.argv[1], **{"%%s_%%d" %% c: T._kout_case(*c) for c in T.KOUT})
print("CHILD_OK")
""" % HERE


@pytest.fixture(scope="module")
def gather_form(tmp_path_factory):
    path = str(tmp_path_factory.mktemp("kout") / "gather.npz")
    env = dict(os.environ, KVQ_KOUT_DIRECT_NPOS=str(1 << 40))
    r = subprocess.run([sys.executable, "-c", CHILD, path], env=env, capture_output=True, text=True, timeout=900,
                       cwd=HERE)
    assert r.returncode == 0 and "CHILD_OK" in r.stdout, (r.stdout[-2000:], r.stderr[-2000:])
    return dict(np.load(path))


@pytest.mark.parametrize("name,j", KOUT)
def test_computed_outlier_factors_equal_the_gather_form(name, j, gather_form):
    got = _kout_case(name, j)
    want = gather_form["%s_%d" % (name, j)]
    assert np.array_equal(got.view(np.uint32), want.view(np.uint32)), int((got != want).sum())


# ---- attends against float64 ------------------------------------------------------------------------------------------
LENGTHS = (1, 33, 8191, 8193, 12000)


@pytest.mark.parametrize("name", sorted(SPECS))
@pytest.mark.parametrize("mode", ["kv", "k", "dense"])
@pytest.mark.parametrize("Hq,Hkv", [(32, 32), (32, 8)])
@pytest.mark.parametrize("bits", [4, 3, 2])
def test_attend_against_float64(bits, Hq, Hkv, mode, name):
    spec = SPECS[name]
    lc = G._cache(bits, Hq, Hkv, mode, Lmax=12004, n_sink=3)
    lc.append_chunk(*G._tokens(lc, max(LENGTHS), seed=bits * 100 + Hq))
    for L in LENGTHS:
        lc.len = L
        q = rotate_q(spec, G._query(Hq, L), lc.n_sink + L)
        for sinks in (False, True):
            lc.sink_k = lc.sink_v = None
            if sinks:
                G._sinks(lc, 3, seed=L)
            out, lse = torch.empty((Hq, 128), device=DEV), torch.empty(Hq, device=DEV)
            lc.attend(q, out=out, lse=lse, rope=spec)
            G._check((out, lse), oracle(lc, q, spec), "L=%d sinks=%s" % (L, sinks))
            if sinks:   # the device-resident length
                out2, lse2 = torch.empty_like(out), torch.empty_like(lse)
                lc.attend_dyn(q, torch.full((1,), L, dtype=torch.int64, device=DEV), 0, out=out2, lse=lse2,
                              L_cap=12000, rope=spec)
                G._check((out2, lse2), oracle(lc, q, spec), "dyn L=%d" % L)
    lc.len, lc.pos_base = 4096, 126 * 1024       # a 4K cache near position 128K
    q = rotate_q(spec, G._query(Hq, 7), lc.n_sink + lc.pos_base + 4096)
    out, lse = torch.empty((Hq, 128), device=DEV), torch.empty(Hq, device=DEV)
    lc.attend(q, out=out, lse=lse, rope=spec)
    want = oracle(lc, q, spec)
    G._check((out, lse), want, "pos_base")
    plain = lc.attend(q, rope_theta=spec.theta).cpu().numpy()   # unscaled: far outside the tolerance
    assert G._head_err(plain, want[0]) > 100 * G.EXACT_TOL


@pytest.mark.parametrize("paged", [False, True])
@pytest.mark.parametrize("name", sorted(SPECS))
def test_batched_attends_against_float64(name, paged):
    from kvquant_b200 import cache as kc
    spec = SPECS[name]
    bits, Hq, Hkv, B, Lmax = 3, 32, 8, 2, 9920
    tmpl = G._cache(bits, Hq, Hkv, "kv", Lmax=Lmax, n_sink=2)
    klut, vcent = tmpl.klut, tmpl.v_cent
    lens = (8190, 9000)
    if paged:
        pt = kc.PageTable(B, 160, 2 * Lmax // 160, Lmax // 160, DEV)
        bc = kc.PagedLayerCache(B, bits, Hkv, klut, None, tmpl.thr_lower, tmpl.thr_upper, vcent, DEV, True, 0.99, 2,
                                None, True, Hq, pages=pt)
    else:
        bc = kc.BatchedLayerCache(B, bits, Hkv, Lmax, klut, None, tmpl.thr_lower, tmpl.thr_upper, vcent, DEV, True,
                                  0.99, 2, None, True, Hq)
    g = torch.Generator(device=DEV).manual_seed(3)
    sk = torch.randn((B, Hkv, 128, 2), generator=g, device=DEV).half()
    sv = torch.randn((B, Hkv, 2, 128), generator=g, device=DEV).half()
    bc.set_sinks(sk, sv)
    qs, want = [], []
    for b, L in enumerate(lens):
        k, v = G._tokens(tmpl, L, seed=b)
        if paged:
            bc.append_chunk(b, k, v)
            bc.commit(b)
        else:
            bc.seq(b).append_chunk(k, v)
            bc.commit(b)
        ref = G._cache(bits, Hq, Hkv, "kv", Lmax=Lmax, n_sink=2)
        ref.append_chunk(k, v)
        ref.set_sinks(sk[b], sv[b])
        q = rotate_q(spec, G._query(Hq, b), 2 + L)
        qs.append(q)
        want.append(oracle(ref, q, spec))
    out, lse = torch.empty((B, Hq, 128), device=DEV), torch.empty((B, Hq), device=DEV)
    bc.attend(torch.stack(qs), out=out, lse=lse, rope=spec)
    torch.cuda.synchronize()
    for b in range(B):
        G._check((out[b], lse[b]), want[b], "b=%d" % b)


# ---- dequantise and chunk attends -------------------------------------------------------------------------------------
@pytest.mark.parametrize("name", sorted(SPECS))
def test_dequantize_and_chunk_attends(name):
    spec = SPECS[name]
    lc = G._cache(4, 32, 8, "kv", Lmax=10004, n_sink=0)
    lc.append_chunk(*G._tokens(lc, 9000, seed=1))
    lc.pos_base = 3
    pre, _ = lc.dequantize(0, 9000)
    rot, _ = lc.dequantize(0, 9000, rope=spec)
    c, s = cos_sin64(spec, 3, 9000)                      # [128, L]
    k = pre.double().cpu().numpy()                       # [H, L, 128]
    kr = np.concatenate([-k[..., 64:], k[..., :64]], axis=-1)
    want = k * c.T[None] + kr * s.T[None]
    got = rot.double().cpu().numpy()
    assert np.abs(got - want).max() <= 2.0 ** -9 * np.abs(want).max()
    T = 96
    kc_, vc_ = G._tokens(lc, T, seed=2)
    p0 = lc.n_sink + lc.pos_base + lc.len
    q = torch.stack([rotate_q(spec, G._query(32, i), p0 + i) for i in range(T)])
    a = lc.attend_chunk(q, kc_, vc_, rope=spec)
    b = lc.attend_chunk_fused(q, kc_, vc_, rope=spec)
    # float64 causal attention over the fp16 operands both chunk attends use
    cc, ss = cos_sin64(spec, p0, T)
    kn = kc_.view(T, 8, 128).double().cpu().numpy()
    knr = np.concatenate([-kn[..., 64:], kn[..., :64]], axis=-1)
    kchunk = (kn * cc.T[:, None] + knr * ss.T[:, None]).astype(np.float16).astype(np.float64).transpose(1, 0, 2)
    K = np.concatenate([got, kchunk], 1)                      # [8, L+T, 128]
    _, vpre = lc.dequantize(0, 9000)
    V = np.concatenate([vpre.double().cpu().numpy(), vc_.view(T, 8, 128).half().double().cpu().numpy().transpose(1, 0, 2)], 1)
    qn = q.half().double().cpu().numpy()                                      # [T, 32, 128]
    S = np.einsum("thc,hsc->ths", qn, np.repeat(K, 4, axis=0)) / np.sqrt(128.0)
    mask = np.arange(9000 + T)[None, :] <= (9000 + np.arange(T))[:, None]
    S = np.where(mask[:, None, :], S, -np.inf)
    P = np.exp(S - S.max(-1, keepdims=True))
    O = np.einsum("ths,hsc->thc", P, np.repeat(V, 4, axis=0)) / P.sum(-1)[..., None]
    scale = np.abs(O).max()
    for got in (a, b):
        assert np.abs(got.double().cpu().numpy() - O).max() <= 2e-3 * scale


def test_default_spec_is_bit_identical_to_theta():
    # K outliers only: the V outlier pass adds with atomics in no fixed order, so two identical calls may differ
    lc = G._cache(3, 32, 8, "k", Lmax=20004, n_sink=2)
    lc.append_chunk(*G._tokens(lc, 20000, seed=5))
    G._sinks(lc, 2, seed=1)
    q = G._query(32, 3)
    for spec in (RotarySpec(10000.0), RotarySpec(10000.0, {"rope_type": "default"})):
        assert torch.equal(lc.attend(q, rope=spec).clone(), lc.attend(q, rope_theta=10000.0).clone())
        a, _ = lc.dequantize(0, 20000, rope=spec)
        b, _ = lc.dequantize(0, 20000, rope_theta=10000.0)
        assert torch.equal(a, b)


# ---- the decode harness -----------------------------------------------------------------------------------------------
def _stage(n_layers=2, max_len=2048):
    from kvquant_b200 import cache as kc, decode as kd, synth
    cfg = kd.DecodeConfig.llama31_8b(n_layers=n_layers, max_len=max_len, n_sink=2)
    sp = synth.SynthSpec(8, 128, seed=0)
    cal = synth.calibrate(sp, 4, calib_tokens=256, seed=7)
    t = kc.build_k_lookup_table(cal["k"][0], cal["k"][1], cal["k"][2][0], 8, device=DEV)
    quant = dict(klut=dict(lut=t["lut"], lut2=None, thr_lower=t["thr_lower"], thr_upper=t["thr_upper"]),
                 v_cent=cal["v"][2][0])
    return kd.DecoderStage(cfg, 0, n_layers, DEV, quant, seed=1, with_head=True)


def test_llama31_stage_prefills_then_decodes_in_one_graph():
    from kvquant_b200 import decode as kd
    st = _stage()
    assert st.rotary == kd.DecodeConfig.llama31_8b().rotary and st.rotary.scaled
    toks = torch.randint(0, st.cfg.vocab, (900,), generator=torch.Generator().manual_seed(0)).to(DEV)
    st.prefill(st.embed[toks], chunk=384)
    L = st.layers[0].cache.len
    gs = kd.GraphedStage(st, L, first=True, last_to_logits=True, dynamic=True)
    steps = [int(x) for x in torch.randint(0, st.cfg.vocab, (8,), generator=torch.Generator().manual_seed(1))]
    got = []
    for tok in steps:
        gs.tok.fill_(tok)
        gs.replay()
        torch.cuda.synchronize()
        got.append(gs.logits.clone())
    st.dyn = None
    st.set_len(L)
    for i, tok in enumerate(steps):
        ref = st.head(st.forward_torch(st.embed_token(torch.tensor([tok], device=DEV))))
        d = (ref.float() - got[i].float()).abs().max().item()
        assert torch.isfinite(got[i].float()).all() and d <= 1e-2 * max(1.0, ref.float().abs().max().item()), (i, d)


def test_llama31_paged_batched_graph_and_forked_prefill():
    from kvquant_b200 import decode as kd
    st = _stage(max_len=1600)
    gen = torch.Generator().manual_seed(2)
    p0, suffix = (torch.randint(0, st.cfg.vocab, (n,), generator=gen).to(DEV) for n in (300, 50))
    toks = torch.randint(0, st.cfg.vocab, (6, 2), generator=gen)
    bst = kd.BatchedDecoderStage(st, 2, page_size=160, n_pool=24)
    bst.prefill_seq(0, st.embed[p0], chunk=256)
    bst.fork_seq(0, 1)
    bst.prefill_seq(1, st.embed[suffix], chunk=64)
    g = kd.BatchedGraphedStep(bst)
    got = []
    for i in range(6):
        g.tok.copy_(toks[i].to(DEV))
        g.replay()
        torch.cuda.synchronize()
        got.append(g.logits.float().clone())
    for b, hist in ((0, [p0]), (1, [p0, suffix])):
        st.set_len(0)
        for h in hist:
            st.prefill(st.embed[h], chunk=256 if h is p0 else 64)
        for i in range(6):
            ref = st.head(st.forward_torch(st.embed_token(toks[i, b:b + 1].to(DEV)))).float()
            d = (ref - got[i][b]).abs().max().item()
            assert torch.isfinite(got[i][b]).all() and d <= 1e-2 * max(1.0, ref.abs().max().item()), (b, i, d)
