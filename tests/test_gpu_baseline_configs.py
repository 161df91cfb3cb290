"""GPU: parity at BASELINE.json's config sizes against the REFERENCE's own CUDA kernels.

  configs[0]  single layer, 4-bit, 4K tokens, with and without 1 % outliers
  configs[1]  LLaMA-7B shapes, 4-bit + 1 % outliers, 32K tokens
  13B shapes  (H = 40, 52 outlier columns), 3-bit, 8K tokens  -- the shape of configs[4] at a size the reference op
              chain finishes in milliseconds

Caches are filled by the real prefill packers (synth.fill_layer_cache_gpu) from seeded inputs; the reference's results
on the same caches are stored in tests/golden/ref_test_gpu_baseline_configs.npz (tests/_refgold.py: a seeded sample of
every head's elements plus every head's largest value; KVQ_REF_GOLDEN_OUT=<dir> compares against the live reference
extension instead and re-records the file):
  * our legacy K / V ops vs the reference's kernels: norm-wise <= 2e-5 AND per head (every head relative to that head's
    own largest value) <= 1e-4 -- a wrong small element cannot hide behind a large one in another head;
  * the fused attend (exact tables, the default) vs the reference op chain K op -> softmax -> V op: <= 1e-4 / per head
    3e-4; with fp16 tables: <= 2e-3 / per head 1e-2 (DESIGN.md section 5 for where that error comes from).
The V op is compared on seeded softmax weights of its own, so that its inputs do not depend on the K op's results."""
import numpy as np
import pytest
import torch

from _refgold import RefGolden, rel_rows

pytestmark = pytest.mark.gpu
DEV = "cuda:0"

CASES = [  # (name, bits, H, L, sparse)
    ("configs0-4b-4k-dense", 4, 32, 4096, False),
    ("configs0-4b-4k-sparse", 4, 32, 4096, True),
    ("configs1-7b-4b-32k", 4, 32, 32768, True),
    ("13b-3b-8k", 3, 40, 8192, True),
]


@pytest.fixture(scope="module")
def gold():
    g = RefGolden("test_gpu_baseline_configs")
    yield g
    g.save()


@pytest.mark.parametrize("name,bits,H,L,sparse", CASES, ids=[c[0] for c in CASES])
def test_ops_and_fused_attend_vs_reference_kernels(gold, name, bits, H, L, sparse):
    from kvquant_b200 import synth, cache as kc, quant_cuda as qc
    sp = synth.SynthSpec(H, 128, seed=0)
    cal = synth.calibrate(sp, bits, calib_tokens=512, seed=7)
    klut = kc.build_k_lookup_table(cal["k"][0], cal["k"][1], cal["k"][2][0], H, device=DEV)
    lc = kc.LayerCache.from_luts(bits, H, L + 64, dict(lut=klut["lut"], lut2=None, thr_lower=klut["thr_lower"],
                                                      thr_upper=klut["thr_upper"]), cal["v"][2][0], device=DEV,
                                 include_sparse=sparse)
    synth.fill_layer_cache_gpu(lc, sp, L, seed=bits + H)
    g = torch.Generator(device=DEV).manual_seed(L + H)
    q = torch.randn((1, H, 128), generator=g, device=DEV).half().float()
    pv = torch.softmax(torch.randn((1, H, L), generator=g, device=DEV) * 2, -1).contiguous()
    lutK = lc.klut.view(H, 128, -1)
    sfx = "2" if sparse else ""
    kname = "vecquant%dmatmul_nuq_perchannel_transposed_rope_mha_batched_fused_opt%s" % (bits, sfx)
    vname = "vecquant%dmatmul_nuq_perchannel_transposed_mha_batched_fused_opt%s" % (bits, sfx)

    def k_op(mod):
        mul = torch.zeros((1, H, L), device=DEV)
        if sparse:
            getattr(mod, kname)(q, lc.kcache, mul, lutK, L, lc.k_outliers, lc.k_outlier_idx, 10000.0, 0)
        else:
            getattr(mod, kname)(q, lc.kcache, mul, lutK, L, 10000.0, 0)
        return mul[0]

    def v_op(mod, p):
        mul = torch.zeros((1, H, 128), device=DEV)
        if sparse:
            getattr(mod, vname)(p, lc.vcache, mul, lc.vlut, L, lc.v_outliers, lc.v_outlier_idx)
        else:
            getattr(mod, vname)(p, lc.vcache, mul, lc.vlut, L)
        return mul[0]

    def ref_chain():
        s_ref = k_op(gold.ref)
        return v_op(gold.ref, torch.softmax(s_ref / np.sqrt(128), -1)[None].contiguous())

    n, h = rel_rows(*gold.rows(name + "/k_op", k_op(qc), lambda: k_op(gold.ref), cols=64))
    assert n < 2e-5 and h < 1e-4, (n, h)
    n, h = rel_rows(*gold.rows(name + "/v_op", v_op(qc, pv), lambda: v_op(gold.ref, pv)))
    assert n < 2e-5 and h < 1e-4, (n, h)
    for precision, tol, tol_head in (("fp32", 1e-4, 3e-4), ("fp16", 2e-3, 1e-2)):
        lc.precision = precision
        fused = lc.attend(q[0].contiguous()).clone()
        n, h = rel_rows(*gold.rows(name + "/chain", fused, ref_chain))
        assert n < tol and h < tol_head, (precision, n, h)
