"""GPU: our ops against the REFERENCE's own CUDA extension on the same inputs.

The reference (deployment/kvquant/quant_cuda.cpp + quant_cuda_kernel.cu, compiled unmodified by oracle/build_ref.py)
is not part of this repository: its results on these seeded inputs are stored in tests/golden/ref_test_gpu_vs_reference.npz
(tests/_refgold.py: digests of the results compared bit for bit, seeded samples of the toleranced ones).  With the
extension built, KVQ_REF_GOLDEN_OUT=<dir> compares against the live reference and re-records the file.

Bars: packed codes / returned index arrays bit-exact; fp32 element-wise outputs bit-exact; matvecs within 2e-5
norm-wise (both sides accumulate in fp32, in different orders; the reference's own order is non-deterministic).
Reference defects are avoided, not reproduced: the 3-bit V prefill packer (quant_cuda_kernel.cu:2574-2579) and the
racy K prefill packer (1857-1883) are compared through the single-token ops instead.
"""
import numpy as np
import pytest
import torch

from _refgold import RefGolden, rel_rows
from _util import O, quantizer, spec

pytestmark = pytest.mark.gpu
DEV = "cuda:0"


@pytest.fixture(scope="module")
def gold():
    g = RefGolden("test_gpu_vs_reference")
    yield g
    g.save()


def cu(x):
    return torch.from_numpy(np.ascontiguousarray(x)).to(DEV)


def _ours(name):
    import quant_cuda
    return getattr(quant_cuda, name)


def _ref(gold, name):
    return getattr(gold.ref, name)


def _close(gold, key, ours, ref_fn, tol=2e-5):
    a, b, bmax = gold.rows(key, ours[0], ref_fn)
    assert rel_rows(a, b, bmax)[0] < tol, (key, rel_rows(a, b, bmax))


@pytest.mark.parametrize("bits", [4, 3, 2])
def test_single_token_appends_bit_exact_vs_reference(gold, bits):
    klut, vcent = quantizer(bits)
    sp = spec()
    H, W, Lmax, T = 32, 128 * bits // 32, 64, 9
    k, v = sp.k_tokens(T, 41), sp.v_tokens(T, 42)
    lut = cu(klut["lut"].reshape(H, 128, -1))
    lo, hi = cu(klut["thr_lower"]), cu(klut["thr_upper"])
    caches = [torch.zeros((H, W, Lmax), dtype=torch.int32, device=DEV) for _ in range(8)]
    vlut = torch.zeros((Lmax, 2 ** bits), dtype=torch.float32, device=DEV)
    ops = ["vecquant%dappendvecK", "vecquant%dappendvecKsparse", "vecquant%dappendvecV", "vecquant%dappendvecVsparse"]
    # even caches: ours; odd caches: the reference's (recording only)
    for t in range(T):
        kv, vv = cu(k[t]), cu(v[t])
        thi, tlo, _, _ = O.v_thresholds(v[t], 21)
        lt = O.v_token_lut(vcent, thi, tlo)
        vlut[t] = cu(lt)
        zp = float(lt[O.zero_point_code(bits)])
        r1, r2 = kv.clone(), kv.clone()
        for i, op in ((0, _ours), (1, lambda n: _ref(gold, n))) if gold.recording else ((0, _ours),):
            op(ops[0] % bits)(caches[i], lut, kv, t)
            op(ops[1] % bits)(caches[2 + i], lut, kv, (r1, r2)[i], lo, hi, t)
            op(ops[2] % bits)(caches[4 + i], vlut, vv, t)
            op(ops[3] % bits)(caches[6 + i], vlut, vv, zp, float(tlo), float(thi), t)
        gold.exact("b%d/rescaled%d" % (bits, t), r1, lambda: r2)
    for i in range(0, 8, 2):
        gold.exact("b%d/%s" % (bits, ops[i // 2] % bits), caches[i], lambda: caches[i + 1])


@pytest.mark.parametrize("bits", [4, 2])
def test_prefill_v_packer_bit_exact_vs_reference(gold, bits):
    # (3-bit is excluded: the reference kernel indexes the LUT by channel there, quant_cuda_kernel.cu:2574-2579)
    klut, vcent = quantizer(bits)
    sp = spec()
    H, W, Lmax, T = 32, 128 * bits // 32, 320, 300
    v = sp.v_tokens(T, 43)
    lo = np.zeros(T, np.float32); hi = np.zeros(T, np.float32)
    vlut = np.zeros((Lmax, 2 ** bits), np.float32)
    for t in range(T):
        hi[t], lo[t], _, _ = O.v_thresholds(v[t], 21)
        vlut[t] = O.v_token_lut(vcent, hi[t], lo[t])
    name = "vecquant%dappendvecVsparseParallel" % bits
    c1 = torch.zeros((H, W, Lmax), dtype=torch.int32, device=DEV)
    c2 = torch.zeros_like(c1)
    vin = cu(v.T.reshape(H, 128, T))
    _ours(name)(c1, cu(vlut), vin, cu(lo), cu(hi))
    gold.exact(name, c1, lambda: (_ref(gold, name)(c2, cu(vlut), vin, cu(lo), cu(hi)), c2)[1])


@pytest.mark.parametrize("bits", [4, 3, 2])
def test_matvecs_vs_reference_kernels(gold, bits):
    from _util import oracle_cache
    L = 700
    c, k, v = oracle_cache(bits, L)
    H, W = 32, 128 * bits // 32
    kc, vc = cu(c.kwords.reshape(H, W, c.Lmax)), cu(c.vwords.reshape(H, W, c.Lmax))
    lut = cu(c.klut["lut"].reshape(H, 128, -1))
    q = cu(O.rope_rotate_q(spec().q_vec(7), L + 3, 10000.0)[None])
    g = torch.Generator(device=DEV).manual_seed(700 + bits)
    p = torch.softmax(torch.randn((1, H, L), generator=g, device=DEV) * 2, -1).half().float()
    for sparse in (False, True):
        sfx = "2" if sparse else ""
        name = "vecquant%dmatmul_nuq_perchannel_transposed_rope_mha_batched_fused_opt%s" % (bits, sfx)
        kargs = (L, cu(c.k_out), cu(c.k_idx), 10000.0, 3) if sparse else (L, 10000.0, 3)

        def k_op(op):
            m = torch.zeros((1, H, L), device=DEV)
            op(q, kc, m, lut, *kargs)
            return m
        _close(gold, name, k_op(_ours(name)), lambda: k_op(_ref(gold, name)))
        name = "vecquant%dmatmul_nuq_perchannel_transposed_mha_batched_fused_opt%s" % (bits, sfx)
        vargs = (L, cu(c.v_out), cu(c.v_idx)) if sparse else (L,)

        def v_op(op):
            o = torch.zeros((1, H, 128), device=DEV)
            op(p, vc, o, cu(c.vlut), *vargs)
            return o
        _close(gold, name, v_op(_ours(name)), lambda: v_op(_ref(gold, name)))


def test_uncapped_orig_path_vs_reference(gold):
    """vecquant4appendvec{K,V}sparseorig + ..._opt2_orig: CSR/CSC arrays and results identical to the reference."""
    import quant_cuda
    klut, vcent = quantizer(4)
    sp = spec()
    H, W, Lmax, T = 32, 16, 64, 12
    k, v = sp.k_tokens(T, 51), sp.v_tokens(T, 52)
    lut = cu(klut["lut"].reshape(H, 128, -1))
    lo, hi, zp = cu(klut["thr_lower"]), cu(klut["thr_upper"]), cu(klut["zeropoint"])
    st = {}
    for name, mod in (("ours", quant_cuda), ("ref", gold.ref)) if gold.recording else (("ours", quant_cuda),):
        kc = torch.zeros((H, W, Lmax), dtype=torch.int32, device=DEV)
        vc = torch.zeros_like(kc)
        vlut = torch.zeros((Lmax, 16), dtype=torch.float32, device=DEV)
        e = lambda: torch.tensor([]).to(DEV)
        rows, cols, vals, start = e(), e(), e(), e()
        vrows, vcols, vvals, vstart = e(), e(), e(), e()
        for t in range(T):
            rows, cols, vals, start, nth, cnt = mod.vecquant4appendvecKsparseorig(kc, lut, cu(k[t]), zp, rows, cols, vals, start, lo, hi, t)
            thi, tlo, _, _ = O.v_thresholds(v[t], 21)
            lt = O.v_token_lut(vcent, thi, tlo)
            vlut[t] = cu(lt)
            vrows, vcols, vvals, vstart, vnth, vcnt = mod.vecquant4appendvecVsparseorig(
                vc, vlut, cu(v[t]), float(lt[7]), vrows, vcols, vvals, vstart, float(tlo), float(thi), t)
        L = T
        q = cu(O.rope_rotate_q(sp.q_vec(3), L, 10000.0)[None])
        mul = torch.zeros((1, H, L), device=DEV)
        mod.vecquant4matmul_nuq_perchannel_transposed_rope_mha_batched_fused_opt2_orig(
            q, kc, mul, lut, L, rows, cols, start, vals, L, int(nth[0]), int(vals.shape[0]), 10000.0, 0)
        p = torch.softmax(torch.arange(H * L, device=DEV).float().view(1, H, L).sin(), -1)
        out = torch.zeros((1, H, 128), device=DEV)
        mod.vecquant4matmul_nuq_perchannel_transposed_mha_batched_fused_opt2_orig(
            p, vc, out, vlut, L, vrows, vcols, vstart, vvals, L, int(vnth[0]), int(vvals.shape[0]))
        st[name] = dict(kc=kc, vc=vc, rows=rows, cols=cols, vals=vals, start=start, nth=int(nth[0]), vrows=vrows,
                        vcols=vcols, vvals=vvals, vstart=vstart, vnth=int(vnth[0]), mul=mul, out=out)
    a, b = st["ours"], st.get("ref")
    for key in ("kc", "vc", "rows", "cols", "vals", "start", "vrows", "vcols", "vvals", "vstart"):
        gold.exact("orig/" + key, a[key], lambda: b[key])
    assert list(gold.value("orig/nth", lambda: [b["nth"], b["vnth"]])) == [a["nth"], a["vnth"]]
    _close(gold, "orig/mul", a["mul"], lambda: b["mul"])
    _close(gold, "orig/out", a["out"], lambda: b["out"])
