"""GPU: the reference's caller code against the drop-in boundary and the repository's mirror classes.

The reference's callers of the `quant_cuda` boundary are `QuantK` / `QuantV` of its modeling_llama.py (lines 352-975,
978-1385).  They are not part of this repository: oracle/build_ref_py.py cuts them verbatim into the git-ignored
oracle/_ref/ref_cache_managers.py when the reference is at hand, and a run with KVQ_REF_GOLDEN_OUT=<dir> (and the
reference extension built, oracle/build_ref.py) drives them through the reference's own sequence -- load_lookup_table,
one prefill `parallel_pack`, then decode steps of `forward_fused_sparse` chained as modeling_llama.py:1803-1820 and
1963-1999 do (CPU top-k of v, scores.half()/sqrt(d), fp32 softmax -> fp16, V op) -- once on the reference's own
extension and once on this repository's shim (kvquant_b200.quant_cuda over the C ABI), and records what they computed
into tests/golden/ref_test_gpu_reference_callers.npz (tests/_refgold.py).

The repository's mirror classes (kvquant_b200.cache.QuantK / QuantV) are driven through the same sequence and compared
with those results: cache words, per-token LUT rows, outlier rows and indices bit for bit (digests); the fp16 scores
and outputs to fp16 accuracy (a seeded sample of every decode step)."""
import math
import os
import sys
import warnings

import numpy as np
import pytest
import torch

from _refgold import RefGolden
from _util import spec, synth

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
DEV = "cuda:0"
H, HID = 32, 4096


@pytest.fixture(scope="module")
def gold():
    g = RefGolden("test_gpu_reference_callers")
    g.mods = None
    if g.recording:
        sys.path.insert(0, os.path.join(ROOT, "oracle"))
        import build_ref_py
        from kvquant_b200 import quant_cuda as shim
        assert os.path.exists(build_ref_py.OUT), "oracle/_ref/ref_cache_managers.py not extracted"
        with warnings.catch_warnings():
            warnings.simplefilter("ignore")
            on_shim = build_ref_py.load(shim, "ref_managers_on_shim")
            on_ref = build_ref_py.load(g.ref, "ref_managers_on_ref")
        assert on_shim.quant_cuda is shim and on_ref.quant_cuda is g.ref
        g.mods = (on_shim, on_ref)
    yield g
    g.save()


def _topk_v(v_flat_gpu, kk):
    """modeling_llama.py:1813-1820: top-k of the new value vector on the CPU, results back on the device."""
    v = v_flat_gpu.cpu()
    uv, ui = torch.topk(v, kk)
    lv, li = torch.topk(v, kk, largest=False)
    return uv.cuda(), ui.cuda(), lv.cuda(), li.cuda()


def _drive(QK, QV, bits, cal, k_pre, v_pre, k_dec, v_dec, q_dec, Lmax):
    """One manager pair through prefill + decode; returns (kmgr, vmgr, scores list, outputs list)."""
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")   # the reference wraps tensors in torch.tensor(...)
        kmgr = QK(bits=bits, hidden_size=HID, num_heads=H, max_position_embeddings=Lmax, include_sparse=True,
                  sparsity_threshold=0.99, rope_theta=10000)
        vmgr = QV(bits=bits, hidden_size=HID, num_heads=H, max_position_embeddings=Lmax, include_sparse=True,
                  sparsity_threshold=0.99)
        kmgr.load_lookup_table(cal["k"], include_sparse=True, sparsity_threshold=0.99)
        vmgr.load_lookup_table(cal["v"], include_sparse=True, sparsity_threshold=0.99)
        kk = int(((1 - 0.99) / 2) * HID) + 2
        T = k_pre.shape[0]
        # prefill (modeling_llama.py:1829-1832, 1907-1927): key_states[0].transpose(1, 2) is [H, 128, T]
        ks = k_pre.view(1, T, H, 128).transpose(1, 2).half()
        vs = v_pre.view(1, T, H, 128).transpose(1, 2).half()
        vf = v_pre.float()
        uv, ui = torch.topk(vf, kk, dim=-1)
        lv, li = torch.topk(vf, kk, dim=-1, largest=False)
        kmgr.parallel_pack(ks[0].transpose(1, 2))
        vmgr.parallel_pack(vs[0].transpose(1, 2), uv, ui, lv, li)
        scores, outs = [], []
        for i in range(k_dec.shape[0]):
            q = q_dec[i].view(H, 1, 128).half()
            kn = k_dec[i].view(1, H, 1, 128).half()
            vn = v_dec[i].view(1, H, 1, 128).half()
            tk = _topk_v(vn.flatten().float(), kk)
            s = kmgr.forward_fused_sparse(q, kn)                               # [H, 1, L] fp16
            scores.append(s.clone())
            a = s.unsqueeze(0) / math.sqrt(128)
            p = torch.nn.functional.softmax(a, dim=-1, dtype=torch.float32).to(torch.float16).squeeze(0)
            o = vmgr.forward_fused_sparse(p, vn, *tk)                          # [H, 1, 128] fp16
            outs.append(o.clone())
    return kmgr, vmgr, scores, outs


def _compare(gold, pre, ours, ref_fn, L, k_lo=0, v_lo=0, fp16_results=True):
    """ours / ref_fn(): (kmgr, vmgr, scores, outs) of two drives; state bit for bit, results to fp16 accuracy."""
    memo = []

    def ref(i):
        if not memo:
            memo.append(ref_fn())
        return memo[0][i]
    ka, va, sa, oa = ours
    gold.exact(pre + "kcache", ka.kcache[:, :, k_lo:L], lambda: ref(0).kcache[:, :, k_lo:L])
    gold.exact(pre + "k_outlier_indices", ka.outlier_indices[k_lo:L], lambda: ref(0).outlier_indices[k_lo:L])
    gold.exact(pre + "k_outliers", ka.outliers[k_lo:L], lambda: ref(0).outliers[k_lo:L])
    gold.exact(pre + "vcache", va.vcache[:, :, v_lo:L], lambda: ref(1).vcache[:, :, v_lo:L])
    gold.exact(pre + "v_lookup_table", va.lookup_table[:L], lambda: ref(1).lookup_table[:L])
    gold.exact(pre + "v_outlier_indices", va.outlier_indices[:L], lambda: ref(1).outlier_indices[:L])
    gold.exact(pre + "v_outliers", va.outliers[:L], lambda: ref(1).outliers[:L])
    if not fp16_results:
        return
    # step i scores [H, 1, L - n + 1 + i]: zero-padded to [H, L] per step, so that they stack to [decode steps, H * L]
    n = len(sa)
    pad = lambda xs: torch.stack([torch.nn.functional.pad(x.float()[:, 0], (0, L - x.shape[-1])).flatten() for x in xs])
    s1, s2, smax = gold.rows(pre + "scores", pad(sa), lambda: pad(ref(2)))
    # fp16 scores: the fp32 results agree to ~1e-6, so at most an occasional one-ulp rounding flip
    d = (s1 - s2).abs().amax(dim=1)
    assert (d <= 2.0 ** -10 * smax.clamp_min(1.0)).all(), d.max().item()
    tok = torch.from_numpy(gold.data[pre + "scores#idx"].astype(np.int64)) % L
    real = tok[None, :] < (L - n + 1 + torch.arange(n))[:, None]       # sampled entries that are not padding
    # at most an occasional flip: the share of equal scores over all sampled (real) entries of all steps
    assert ((s1 == s2) & real).sum() > 0.98 * real.sum(), (((s1 == s2) & real).sum().item(), real.sum().item())
    stack = lambda xs: torch.stack([x.float().flatten() for x in xs])   # [decode steps, H * 128]
    o1, o2, omax = gold.rows(pre + "outs", stack(oa), lambda: stack(ref(3)))
    d = (o1 - o2).abs().amax(dim=1)
    assert (d <= 2e-3 * omax.clamp_min(1e-3)).all(), d.max().item()


@pytest.mark.parametrize("bits", [4, 3])
def test_reference_quantk_quantv_run_unmodified_on_the_shim(gold, bits):
    """The mirror classes on the shim reproduce the reference's classes on the reference's own extension."""
    from kvquant_b200 import cache as kc
    sp = spec()
    cal = synth.calibrate(sp, bits, calib_tokens=512, seed=7)
    # prefill of 32 tokens: the reference's K prefill packer stages its tables in shared memory without a barrier
    # (quant_cuda_kernel.cu:1857-1883; 128 threads per block); with more than one warp of tokens its output is not
    # reproducible run to run, so a bit-for-bit comparison against it is only meaningful while one warp owns all the
    # tokens.  When even that disagreed with itself while recording, only the decode-time K slots are compared.
    T, ND = 32, 64
    Lmax = 256
    k_all = torch.from_numpy(sp.k_tokens(T + ND, seed=21)).to(DEV)
    v_all = torch.from_numpy(sp.v_tokens(T + ND, seed=22)).to(DEV)
    # fp16-representable inputs: the reference feeds .half() activations to both managers
    k_all, v_all = k_all.half().float(), v_all.half().float()
    g = torch.Generator(device=DEV).manual_seed(5)
    q_dec = torch.randn((ND, H, 128), generator=g, device=DEV)
    args = (bits, cal, k_all[:T], v_all[:T], k_all[T:], v_all[T:], q_dec, Lmax)
    ours = _drive(kc.QuantK, kc.QuantV, *args)
    L = T + ND
    assert ours[0].klen == L and ours[1].vlen == L
    ref_runs = []

    def racy():
        on_ref = gold.mods[1]
        ref_runs.extend([_drive(on_ref.QuantK, on_ref.QuantV, *args) for _ in range(2)])
        a, b = ref_runs[0][0], ref_runs[1][0]
        return [not (torch.equal(a.kcache[:, :, :T], b.kcache[:, :, :T]) and torch.equal(a.outliers[:T], b.outliers[:T]))]
    k_lo = T if bool(gold.value("b%d/k_prefill_racy" % bits, racy)[0]) else 0
    # 3-bit V prefill: the reference kernel indexes the LUT by channel for entries 1..7 (quant_cuda_kernel.cu:2574-2579,
    # a defect our packer does not reproduce, DESIGN.md section 2) -> compare V codes from the decode-time slots only,
    # and the V outputs not at all
    v_lo = T if bits == 3 else 0
    _compare(gold, "ref_on_ref/b%d/" % bits, ours, lambda: ref_runs[0], L, k_lo, v_lo, fp16_results=(bits != 3))


@pytest.mark.parametrize("bits", [4, 3, 2])
def test_mirror_classes_equal_the_reference_classes_on_the_shim(gold, bits):
    """kvquant_b200.cache.QuantK / QuantV (device-side top-k, vectorised LUT build) against the reference's own classes,
    both on the shim: same caches bit for bit, same fp16 results (same kernels, same inputs)."""
    from kvquant_b200 import cache as kc
    sp = spec()
    cal = synth.calibrate(sp, bits, calib_tokens=512, seed=7)
    T, ND = 32, 24
    Lmax = 128
    k_all = torch.from_numpy(sp.k_tokens(T + ND, seed=31)).to(DEV).half().float()
    v_all = torch.from_numpy(sp.v_tokens(T + ND, seed=32)).to(DEV).half().float()
    g = torch.Generator(device=DEV).manual_seed(6)
    q_dec = torch.randn((ND, H, 128), generator=g, device=DEV)
    args = (bits, cal, k_all[:T], v_all[:T], k_all[T:], v_all[T:], q_dec, Lmax)
    ours = _drive(kc.QuantK, kc.QuantV, *args)
    memo = []

    def ref():
        if not memo:
            memo.append(_drive(gold.mods[0].QuantK, gold.mods[0].QuantV, *args))
        return memo[0]
    gold.exact("ref_on_shim/b%d/k_lut" % bits, ours[0].lookup_table.view(-1), lambda: ref()[0].lookup_table.view(-1))
    _compare(gold, "ref_on_shim/b%d/" % bits, ours, ref, T + ND)
