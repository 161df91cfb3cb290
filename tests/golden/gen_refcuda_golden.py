#!/usr/bin/env python
"""Generate tests/golden/refcuda_b{4,3,2}.npz from the REFERENCE's own CUDA kernels.

Runs on a GPU: imports oracle/_ref/quant_cuda_ref.so -- the unmodified reference extension
(deployment/kvquant/quant_cuda.cpp + quant_cuda_kernel.cu) compiled by oracle/build_ref.py -- feeds it
seeded synthetic inputs at small sizes and stores inputs + outputs.  The fixtures are committed; the CPU-only test
tests/test_oracle_golden.py::test_kernel_semantics_match_reference_cuda_fixtures pins the numpy oracle to them.

    python tests/golden/gen_refcuda_golden.py [OUT_DIR]      # writes OUT_DIR/refcuda_b*.npz (default: the cwd)
"""
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "oracle"))
sys.path.insert(0, os.path.join(ROOT, "tests"))

import build_ref  # noqa: E402
from _util import O, quantizer, spec  # noqa: E402  (oracle is used only to build inputs: LUTs, thresholds)

DEV = "cuda:0"


def cu(x):
    return torch.from_numpy(np.ascontiguousarray(x)).to(DEV)


def main():
    ref = build_ref.load()
    assert ref is not None, "oracle/_ref/quant_cuda_ref.so missing"
    out_dir = sys.argv[1] if len(sys.argv) > 1 else os.getcwd()
    os.makedirs(out_dir, exist_ok=True)
    sp = spec()
    H, T, Lmax = 32, 16, 32
    for bits in (4, 3, 2):
        klut, vcent = quantizer(bits)
        W = 128 * bits // 32
        k, v = sp.k_tokens(T, 900 + bits), sp.v_tokens(T, 950 + bits)
        lut = cu(klut["lut"].reshape(H, 128, -1))
        lo, hi = cu(klut["thr_lower"]), cu(klut["thr_upper"])
        kc = torch.zeros((H, W, Lmax), dtype=torch.int32, device=DEV)
        vc = torch.zeros_like(kc)
        vlut = torch.zeros((Lmax, 2 ** bits), dtype=torch.float32, device=DEV)
        resc = np.zeros((T, 4096), np.float32)
        thr = np.zeros((T, 2), np.float32)
        k_out = np.zeros((Lmax, 42), np.float32); k_idx = np.zeros((Lmax, 42), np.int32)
        v_out = np.zeros((Lmax, 42), np.float32); v_idx = np.zeros((Lmax, 42), np.int32)
        for t in range(T):
            kv, vv = cu(k[t]), cu(v[t])
            r = kv.clone()
            getattr(ref, "vecquant%dappendvecKsparse" % bits)(kc, lut, kv, r, lo, hi, t)
            resc[t] = r.cpu().numpy()
            # host glue of the reference (ML.py:706-751, 1091-1176) via the oracle's restatement -- inputs to the matvecs
            k_out[t], k_idx[t] = O.k_outlier_row(k[t], resc[t], klut["lut"], 21)
            thi, tlo, ui, li = O.v_thresholds(v[t], 21)
            lt = O.v_token_lut(vcent, thi, tlo)
            vlut[t] = cu(lt)
            thr[t] = (tlo, thi)
            getattr(ref, "vecquant%dappendvecVsparse" % bits)(vc, vlut, vv, float(lt[O.zero_point_code(bits)]), float(tlo), float(thi), t)
            v_out[t], v_idx[t] = O.v_outlier_row(v[t], ui, li, lt[O.zero_point_code(bits)])
        q = O.rope_rotate_q(sp.q_vec(77), T + 2, 10000.0)
        p = O.softmax_f32(np.random.default_rng(bits).standard_normal((H, T)).astype(np.float32)).astype(np.float16).astype(np.float32)
        res = {}
        for name, sparse in (("dense", False), ("sparse", True)):
            mul = torch.zeros((1, H, T), device=DEV)
            kn = "vecquant%dmatmul_nuq_perchannel_transposed_rope_mha_batched_fused_opt%s" % (bits, "2" if sparse else "")
            if sparse:
                getattr(ref, kn)(cu(q[None]), kc, mul, lut, T, cu(k_out), cu(k_idx), 10000.0, 2)
            else:
                getattr(ref, kn)(cu(q[None]), kc, mul, lut, T, 10000.0, 2)
            res["k_scores_" + name] = mul.cpu().numpy()[0]
            o = torch.zeros((1, H, 128), device=DEV)
            vn = "vecquant%dmatmul_nuq_perchannel_transposed_mha_batched_fused_opt%s" % (bits, "2" if sparse else "")
            if sparse:
                getattr(ref, vn)(cu(p[None]), vc, o, vlut, T, cu(v_out), cu(v_idx))
            else:
                getattr(ref, vn)(cu(p[None]), vc, o, vlut, T)
            res["v_out_" + name] = o.cpu().numpy()[0]
        path = os.path.join(out_dir, "refcuda_b%d.npz" % bits)
        np.savez_compressed(path, bits=bits, T=T, Lmax=Lmax, k=k, v=v,
                            kcache=kc.cpu().numpy().reshape(-1, Lmax), vcache=vc.cpu().numpy().reshape(-1, Lmax),
                            rescaled=resc, v_thr=thr, vlut=vlut.cpu().numpy(), q=q, p=p, k_out=k_out, k_idx=k_idx,
                            v_out=v_out, v_idx=v_idx, **res)
        print("wrote", path, os.path.getsize(path))


if __name__ == "__main__":
    main()
