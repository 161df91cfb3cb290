#!/usr/bin/env python
"""Causal attention of a prompt chunk over the quantised cache: LayerCache.attend_chunk_fused (tensor cores, K/V
tiles dequantised in shared memory) against LayerCache.attend_chunk (whole cache dequantised to fp16 in HBM, then
scaled_dot_product_attention).

    python scripts/measure_chunk_attend.py [--lengths 32768 131072] [--chunks 1 64 512 2048] [--calls 7] [--out FILE]

Prints one JSON line:
  * gpu: card name, power limit and maximum SM clock, read in the same run;
  * runs: per shape (LLaMA-7B 4-bit and 3-bit with 1 % K and V outliers, LLaMA-13B 4-bit with 1 %), cache length L and
    chunk length T, the median of `--calls` CUDA-event timings of each method, taken alternately after one warm-up
    call each; the peak extra device memory of one call of each (torch.cuda.max_memory_allocated growth); the flops
    the attention needs, 4*T*H*128*L + 2*T*(T+1)*H*128 (no sinks here), the achieved TFLOP/s and its fraction of the
    H100 SXM data sheet's 989 TFLOP/s dense fp16 (a data-sheet figure, not a measured peak);
  * plus LLaMA-7B 4-bit dense-only at L = 1M, T = 512, the cache filled with random codes and (sf, off).
attend_chunk runs only where its K/V buffers and mask take at most a fifth of the free device memory
(torch.cuda.mem_get_info()); elsewhere it is recorded as skipped with the GiB it would need.
"""
import argparse
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "scripts"))

from measure_dequant import make_caches  # noqa: E402
from measure_wide_heads import gpu_info  # noqa: E402

SHAPES = (("llama7b_4bit", 32, 4), ("llama7b_3bit", 32, 3), ("llama13b_4bit", 40, 4))
PEAK_TFLOPS = 989.0     # H100 SXM data sheet, dense fp16 tensor core


def flops(T, H, L):
    return 4 * T * H * 128 * L + 2 * T * (T + 1) * H * 128


def measure(lc, T, calls, theta, dev):
    import torch
    H = lc.H
    g = torch.Generator(device=dev).manual_seed(T)
    q = torch.randn((T, H, 128), generator=g, device=dev)
    k = torch.randn((T, H * 128), generator=g, device=dev)
    v = torch.randn((T, H * 128), generator=g, device=dev)
    L = lc.len
    S = L + T
    need = 2 * H * S * 128 * 2 + T * S
    free, _ = torch.cuda.mem_get_info(dev)
    methods = {"fused": lambda: lc.attend_chunk_fused(q, k, v, rope_theta=theta)}
    rec = {"tokens": L, "chunk": T, "flops": flops(T, H, L)}
    if need <= free / 5:
        methods["attend_chunk"] = lambda: lc.attend_chunk(q, k, v, rope_theta=theta)
    else:
        rec["attend_chunk"] = {"skipped": True, "gib_needed": need / 2 ** 30, "gib_free": free / 2 ** 30}
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    for name, fn in methods.items():      # warm-up (rope table, allocator, SDPA kernel choice) and peak memory
        fn()
        torch.cuda.synchronize()
        torch.cuda.reset_peak_memory_stats(dev)
        m0 = torch.cuda.memory_allocated(dev)
        fn()
        torch.cuda.synchronize()
        rec[name] = {"peak_extra_bytes": torch.cuda.max_memory_allocated(dev) - m0}
    ms = {name: [] for name in methods}
    for _ in range(calls):
        for name, fn in methods.items():
            a.record()
            fn()
            b.record()
            torch.cuda.synchronize()
            ms[name].append(a.elapsed_time(b))
    for name in methods:
        med = sorted(ms[name])[len(ms[name]) // 2]
        tf = rec["flops"] / med / 1e9
        rec[name].update({"ms": med, "tflops": tf, "frac_of_989": tf / PEAK_TFLOPS})
    if "attend_chunk" in methods:
        rec["fused_speedup"] = rec["attend_chunk"]["ms"] / rec["fused"]["ms"]
        got, want = methods["fused"](), methods["attend_chunk"]()
        rec["max_abs_diff_rel"] = ((got - want).abs().max() / want.abs().max()).item()
    return rec


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--lengths", type=int, nargs="+", default=[32768, 131072])
    ap.add_argument("--chunks", type=int, nargs="+", default=[1, 64, 512, 2048])
    ap.add_argument("--calls", type=int, default=7)
    ap.add_argument("--million", type=int, default=1 << 20, help="length of the dense-only run (0: skip)")
    ap.add_argument("--out", default=None, help="also write the JSON line to this file")
    args = ap.parse_args()

    import torch
    if not torch.cuda.is_available():
        raise SystemExit("needs a CUDA device")
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    theta = 10000.0
    runs = []
    for name, H, bits in SHAPES:
        for L in args.lengths:
            _, (lc,) = make_caches(H, bits, L, 64, dev, n=1)
            for T in args.chunks:
                r = measure(lc, T, args.calls, theta, dev)
                r["shape"] = name
                runs.append(r)
                print(json.dumps(r), file=sys.stderr, flush=True)
            del lc
            torch.cuda.empty_cache()
    if args.million:
        from kvquant_b200 import synth, cache as kc
        H, bits, L = 32, 4, args.million
        cal = synth.calibrate(synth.SynthSpec(H, 128, seed=0), bits, calib_tokens=512, seed=7)
        t = kc.build_k_lookup_table(cal["k"][0], cal["k"][1], cal["k"][2][0], H, device=dev)
        klut = dict(lut=t["lut"], lut2=None, thr_lower=t["thr_lower"], thr_upper=t["thr_upper"])
        lc = kc.LayerCache.from_luts(bits, H, L, klut, cal["v"][2][0], device=dev, include_sparse=False)
        g = torch.Generator(device=dev).manual_seed(5)
        for x in (lc.kcache, lc.vcache):
            x.copy_(torch.randint(-2 ** 31, 2 ** 31, x.shape, generator=g, device=dev, dtype=torch.int64).to(torch.int32))
        lc.vaff[:, 0] = torch.rand(L, generator=g, device=dev) + 0.5
        lc.vaff[:, 1] = torch.rand(L, generator=g, device=dev) - 0.5
        lc.len = L
        r = measure(lc, 512, args.calls, theta, dev)
        r["shape"] = "llama7b_4bit_dense"
        runs.append(r)
        del lc
        torch.cuda.empty_cache()

    line = {"what": "LayerCache.attend_chunk_fused vs attend_chunk, batch 1, one layer, one GPU", "gpu": gpu_info(0),
            "runs": runs, "timing": "median of %d single calls per method (CUDA events), alternating" % args.calls,
            "peak_tflops": PEAK_TFLOPS, "peak_source": "H100 SXM data sheet dense fp16 (989 TFLOP/s), not measured"}
    s = json.dumps(line)
    print(s, flush=True)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            f.write(s + "\n")
    return 0


if __name__ == "__main__":
    sys.exit(main())
