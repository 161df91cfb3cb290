"""GPU: head counts whose native V tile does not fit one CTA's shared memory (4-bit H >= 36, 3-bit H >= 60).

The native score.V pass then splits the heads into two groups, one CTA per (token range, head group).  These tests
cover that form through every entry point that uses it: the host-length attend against the CPU oracle, the
device-resident-length attend against the host-length one, V outliers on both sides of the head-group boundary, the
one-graph decode loop at the LLaMA-13B shape, and a full-size (128K-token) layer against the legacy two-op chain."""
import numpy as np
import pytest
import torch

from _util import O, oracle_cache, quantizer, rel_err, spec

pytestmark = pytest.mark.gpu
DEV = "cuda:0"

# (bits, H): 4-bit H = 40 / 48 / 64 (LLaMA-13B, -, LLaMA-65B), 3-bit H = 60 / 64.  Outlier widths 52 / 62 / 82 / 78 / 82:
# the last three pass 64 columns, the V kernel's unprefetched tail
WIDE = [(4, 40), (4, 48), (4, 64), (3, 60), (3, 64)]


def cu(x):
    return torch.from_numpy(np.ascontiguousarray(x)).to(DEV)


def _appended_cache(bits, H, L):
    """LayerCache filled token by token with the fused device append, checked bit-exact against the oracle cache."""
    from kvquant_b200.cache import LayerCache
    c, k, v = oracle_cache(bits, L, H=H)
    klut, vcent = quantizer(bits, H=H)
    lc = LayerCache.from_luts(bits, H, c.Lmax, klut, vcent, device=DEV)
    kd, vd = cu(k), cu(v)
    for t in range(L):
        lc.append(kd[t], vd[t])
    assert np.array_equal(lc.kcache.cpu().numpy().reshape(-1, c.Lmax), c.kwords)
    assert np.array_equal(lc.vcache.cpu().numpy().reshape(-1, c.Lmax), c.vwords)
    for name, want in (("k_outlier_idx", c.k_idx), ("v_outlier_idx", c.v_idx), ("k_outliers", c.k_out),
                       ("v_outliers", c.v_out)):
        assert np.array_equal(getattr(lc, name).cpu().numpy(), want), name
    return c, lc


@pytest.mark.parametrize("L", [150, 1000])
@pytest.mark.parametrize("bits,H", WIDE)
def test_wide_head_append_and_attend_match_oracle(bits, H, L):
    c, lc = _appended_cache(bits, H, L)
    assert c.k_out.shape[1] == {40: 52, 48: 62, 60: 78, 64: 82}[H]
    q = O.rope_rotate_q(spec(H).q_vec(L + H), L, 10000.0)
    s = c.k_scores(q)
    _, want = O.attend_ideal(s, c.v_output)
    want_o, want_lse = O.attend_partial(s, c.v_output)
    lse = torch.empty(H, device=DEV)
    for precision, tol in (("fp16", 1.5e-3), ("fp32", 1e-3)):
        lc.precision = precision
        out = lc.attend(cu(q), lse=lse).cpu().numpy()
        assert rel_err(out, want)[0] < tol, (precision, rel_err(out, want))
    assert rel_err(out, want_o)[0] < 1e-3
    # log-sum-exp of the exact-table run, relative to its scale: it carries the fp32 rounding of the scores (scaled
    # scores of up to ~|lse|, so a few 1e-6 relative against the float64 oracle at any head count), while a head group
    # whose denominators went missing or were counted twice would be off by O(1)
    assert rel_err(lse.cpu().numpy(), want_lse)[0] < 2e-5, rel_err(lse.cpu().numpy(), want_lse)


@pytest.mark.parametrize("n_sink", [0, 5])
@pytest.mark.parametrize("bits,H", [(4, 40), (3, 64)])
def test_wide_head_device_resident_length_equals_host_length(bits, H, n_sink):
    """kvq_attend_dyn at a head-split shape: several lengths under ONE set of launch parameters (grid sized for the
    whole allocation) give the host-length attend's result."""
    from kvquant_b200.cache import LayerCache
    L = 1000
    c, k, v = oracle_cache(bits, L, H=H)
    klut, vcent = quantizer(bits, H=H)
    sp = spec(H)
    a = LayerCache.from_luts(bits, H, c.Lmax, klut, vcent, device=DEV, n_sink=n_sink)
    b = LayerCache.from_luts(bits, H, c.Lmax, klut, vcent, device=DEV, n_sink=n_sink)
    a.load_state(c)
    b.load_state(c)
    if n_sink:
        g = torch.Generator(device=DEV).manual_seed(H)
        ks = torch.randn((H, 128, n_sink), generator=g, device=DEV).half()
        vs = torch.randn((H, n_sink, 128), generator=g, device=DEV).half()
        a.set_sinks(ks, vs)
        b.set_sinks(ks, vs)
    len_dev = torch.zeros(1, dtype=torch.int64, device=DEV)
    for precision in ("fp32", "fp16"):
        a.precision = b.precision = precision
        for Lt in (L, L // 2 + 3, 33, 1):
            q = cu(O.rope_rotate_q(sp.q_vec(3 + Lt), Lt + n_sink, 10000.0))
            a.len = Lt
            want = a.attend(q).clone()
            len_dev.fill_(Lt - 1)
            got = b.attend_dyn(q, len_dev, 1).clone()
            assert rel_err(got.cpu().numpy(), want.cpu().numpy())[0] < 1e-5, (precision, Lt)


def _v_tokens_loud_in(heads, H, L, seed):
    """V tokens whose large values (and so every V outlier of a token) sit in the channels of `heads`."""
    rng = np.random.default_rng(seed)
    v = rng.standard_normal((L, H * 128)).astype(np.float32) * 0.1
    for h in heads:
        v[:, h * 128:(h + 1) * 128] = rng.standard_normal((L, 128)).astype(np.float32) * 3.0
    return v


@pytest.mark.parametrize("mode", ["kv", "dense", "k_only"])
@pytest.mark.parametrize("heads", [(19, 20), (30, 39)])
def test_v_outliers_at_the_head_group_boundary(heads, mode):
    """H = 40 at 4 bits splits into heads 0-19 and 20-39.  Outliers in heads 19 and 20 straddle the boundary (each CTA
    must apply exactly its own half of every row); in heads 30 and 39 they all belong to group 1 (group 0 applies
    none).  Repeated for a dense-only cache and a K-only outlier cache, where the V side has no rows at all."""
    from kvquant_b200.cache import LayerCache
    bits, H, L, Lmax = 4, 40, 300, 384
    klut, vcent = quantizer(bits, H=H)
    sp = spec(H)
    k = sp.k_tokens(L, seed=51)
    v = _v_tokens_loud_in(heads, H, L, seed=52)
    sparse, sparse_v = mode != "dense", mode == "kv"
    c = O.OracleCache(bits, H, Lmax, klut, vcent, include_sparse=sparse, sparse_v=sparse_v)
    lc = LayerCache.from_luts(bits, H, Lmax, klut, vcent, device=DEV, include_sparse=sparse, sparse_v=sparse_v)
    kd, vd = cu(k), cu(v)
    for t in range(L):
        c.append(k[t], v[t])
        lc.append(kd[t], vd[t])
    assert np.array_equal(lc.vcache.cpu().numpy().reshape(-1, Lmax), c.vwords)
    if sparse_v:
        assert np.array_equal(lc.v_outlier_idx.cpu().numpy(), c.v_idx)
        assert np.array_equal(lc.v_outliers.cpu().numpy(), c.v_out)
        assert set(np.unique(c.v_idx[:L] // 128)) == set(heads)
    q = O.rope_rotate_q(sp.q_vec(6), L, 10000.0)
    _, want = O.attend_ideal(c.k_scores(q), c.v_output)
    # exact tables: what is checked here is the V side (the fp16 K tables are covered above)
    lc.precision = "fp32"
    out = lc.attend(cu(q)).cpu().numpy()
    assert rel_err(out, want)[0] < 1e-3, rel_err(out, want)
    # the loud heads against their own scale: a head missing (or doubling) its outliers would show here
    hs = list(heads)
    d = np.abs(out[hs] - want[hs]).max(axis=1) / np.abs(want[hs]).max(axis=1)
    assert d.max() < 1e-3, d


def test_dynamic_length_graph_decodes_llama13b_shape_at_4_bits():
    """ONE captured graph with the device-resident length (40 heads, 4 bits: the head-split V pass) replayed 4 times
    == 4 eager steps with host lengths."""
    from kvquant_b200 import decode as kd, synth, cache as kc
    L, H = 96, 40
    cfg = kd.DecodeConfig(n_layers=2, hidden=5120, n_heads=H, intermediate=1024, vocab=512, bits=4, n_sink=3,
                          max_len=L + 64)
    sp = synth.SynthSpec(H, 128, seed=0)
    cal = synth.calibrate(sp, cfg.bits, calib_tokens=256, seed=7)
    t = kc.build_k_lookup_table(cal["k"][0], cal["k"][1], cal["k"][2][0], H, device=DEV)
    quant = dict(klut=dict(lut=t["lut"], lut2=None, thr_lower=t["thr_lower"], thr_upper=t["thr_upper"]), v_cent=cal["v"][2][0])
    st = kd.DecoderStage(cfg, 0, cfg.n_layers, DEV, quant, seed=1, with_head=True)
    for i, ly in enumerate(st.layers):
        synth.fill_layer_cache_gpu(ly.cache, sp, L, seed=i, chunk=64)
    gs = kd.GraphedStage(st, L, first=True, last_to_logits=True, dynamic=True)
    toks = [7, 11, 3, 250]
    got = []
    for tok in toks:
        gs.tok.fill_(tok)
        gs.replay()
        torch.cuda.synchronize()
        got.append(gs.logits.clone())
    assert st.layers[0].cache.len == L + len(toks)
    assert int(st.dyn["len"].item()) == L + len(toks)
    st.dyn = None
    st.set_len(L)
    for i, tok in enumerate(toks):
        y = st.forward(st.embed_token(torch.tensor([tok], device=DEV)))
        ref = st.head(y)
        d = (ref.float() - got[i].float()).abs().max().item()
        assert d <= 1e-2 * max(1.0, ref.float().abs().max().item()), (i, d)


def test_llama13b_4bit_full_size_attend_equals_the_two_op_chain():
    """One LLaMA-13B layer at 4 bits, 131072 tokens, 1 % outliers: the head-split V pass together with the 64-bit
    offsets and the direct cos/sin path used beyond 64K positions.  The fused attend (host and device-resident length)
    == the legacy chain K op -> softmax -> V op, whose ops are oracle-checked at small sizes."""
    from kvquant_b200 import synth, cache as kc, quant_cuda as qc
    bits, H, L = 4, 40, 131072
    sp = synth.SynthSpec(H, 128, seed=0)
    cal = synth.calibrate(sp, bits, calib_tokens=512, seed=7)
    t = kc.build_k_lookup_table(cal["k"][0], cal["k"][1], cal["k"][2][0], H, device=DEV)
    lc = kc.LayerCache.from_luts(bits, H, L + 64, dict(lut=t["lut"], lut2=None, thr_lower=t["thr_lower"],
                                                       thr_upper=t["thr_upper"]), cal["v"][2][0], device=DEV)
    synth.fill_layer_cache_gpu(lc, sp, L, seed=13)
    g = torch.Generator(device=DEV).manual_seed(1)
    q = torch.randn((1, H, 128), generator=g, device=DEV).half().float()
    s = torch.zeros((1, H, L), device=DEV)
    qc.vecquant4matmul_nuq_perchannel_transposed_rope_mha_batched_fused_opt2(
        q, lc.kcache, s, lc.klut.view(H, 128, -1), L, lc.k_outliers, lc.k_outlier_idx, 10000.0, 0)
    p = torch.softmax(s[0] / np.sqrt(128), -1)[None].contiguous()
    chain = torch.zeros((1, H, 128), device=DEV)
    qc.vecquant4matmul_nuq_perchannel_transposed_mha_batched_fused_opt2(p, lc.vcache, chain, lc.vlut, L, lc.v_outliers,
                                                                       lc.v_outlier_idx)
    chain = chain[0]
    lc.precision = "fp32"
    fused = lc.attend(q[0].contiguous()).clone()
    len_dev = torch.full((1,), L - 1, dtype=torch.int64, device=DEV)
    dyn = lc.attend_dyn(q[0].contiguous(), len_dev, 1).clone()

    def rel(a, b):
        return ((a - b).abs().max() / b.abs().max()).item()
    assert rel(fused, chain) < 1e-4, rel(fused, chain)
    assert rel(dyn, chain) < 1e-4, rel(dyn, chain)
