#!/usr/bin/env python
"""The quantised cache read back on the device: LayerCache.dequantize and LayerCache.attend_chunk.

    python scripts/measure_dequant.py [--lengths 32768 131072] [--calls 100] [--chunk 512] [--out FILE]

Prints one JSON line:
  * gpu: card name, power limit and maximum SM clock, read in the same run;
  * dequant: per shape (LLaMA-7B 4-bit and 3-bit, LLaMA-13B 4-bit, 1 % K and V outliers) and length, the time of one
    whole-cache dequantize() into preallocated outputs, pre-RoPE and rotated.  Median of `--calls` calls timed one by
    one with CUDA events, alternating between two caches of identical contents (each larger than the 50 MB L2).
    Bytes are computed from the shapes: read = codes (2*hidden*bits/8) + outlier rows (2 * n_out * 8) + (sf, off) (8)
    per token, written = 2*hidden fp16 per token; their sum over the time as GB/s and as a fraction of the H100 SXM
    data sheet's 3.35 TB/s.  The rotated form also reads the shared cos/sin table (512 B per token), not counted;
  * chunk: attend_chunk of `--chunk` tokens after a 32K-token 7B 4-bit cache, against the same tokens handled one at a
    time as decode does today (append + attend per token, on a copy of the cache).
"""
import argparse
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "scripts"))

from measure_wide_heads import CACHE_TENSORS, PEAK_GBS, gpu_info, median_call_ms  # noqa: E402

SHAPES = (("llama7b_4bit", 32, 4), ("llama7b_3bit", 32, 3), ("llama13b_4bit", 40, 4))


def make_caches(H, bits, L, extra, dev, n=2):
    """n LayerCaches of L synthetic tokens (1 % K and V outliers), filled through the prefill packers."""
    from kvquant_b200 import synth, cache as kc
    sp = synth.SynthSpec(H, 128, seed=0)
    cal = synth.calibrate(sp, bits, calib_tokens=512, seed=7)
    t = kc.build_k_lookup_table(cal["k"][0], cal["k"][1], cal["k"][2][0], H, device=dev)
    klut = dict(lut=t["lut"], lut2=None, thr_lower=t["thr_lower"], thr_upper=t["thr_upper"])
    out = [kc.LayerCache.from_luts(bits, H, L + extra, klut, cal["v"][2][0], device=dev) for _ in range(n)]
    synth.fill_layer_cache_gpu(out[0], sp, L, seed=0)
    for lc in out[1:]:
        for name in CACHE_TENSORS:
            getattr(lc, name).copy_(getattr(out[0], name))
        lc.len = L
    return sp, out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--lengths", type=int, nargs="+", default=[32768, 131072])
    ap.add_argument("--calls", type=int, default=100)
    ap.add_argument("--chunk", type=int, default=512)
    ap.add_argument("--out", default=None, help="also write the JSON line to this file")
    args = ap.parse_args()

    import torch
    from kvquant_b200 import quant_cuda as qc
    if not torch.cuda.is_available():
        raise SystemExit("needs a CUDA device")
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    theta = 10000.0

    dequant = []
    for name, H, bits in SHAPES:
        for L in args.lengths:
            _, caches = make_caches(H, bits, L, 64, dev)
            lc = caches[0]
            out_k = torch.empty((H, L, 128), dtype=torch.float16, device=dev)
            out_v = torch.empty_like(out_k)
            qc.rope_tables(dev, theta, L + 1)
            hidden = H * 128
            read = L * (2 * hidden * bits // 8 + 2 * lc.n_out * 8 + 8)
            written = L * 2 * hidden * 2
            rec = {"shape": name, "tokens": L, "bytes_read": read, "bytes_written": written}
            for form, rope in (("prerope", None), ("rotated", theta)):
                ms = median_call_ms(lambda c: c.dequantize(rope_theta=rope, out_k=out_k, out_v=out_v), caches,
                                    args.calls, warm=4)
                gbs = (read + written) / ms / 1e6
                rec[form] = {"ms": ms, "gbs": gbs, "frac_of_3350": gbs / PEAK_GBS}
            dequant.append(rec)
            del caches, lc, out_k, out_v
            torch.cuda.empty_cache()

    # ---- attend_chunk vs one token at a time -----------------------------------------------------------------------
    L, T, H, bits = 32768, args.chunk, 32, 4
    sp, (lc, seq) = make_caches(H, bits, L, T + 64, dev)
    g = torch.Generator(device=dev).manual_seed(3)
    q = torch.randn((T, H, 128), generator=g, device=dev)
    k = torch.randn((T, H * 128), generator=g, device=dev)
    v = torch.randn((T, H * 128), generator=g, device=dev)
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)

    def timed(fn, reps):
        fn()
        torch.cuda.synchronize()
        ms = []
        for _ in range(reps):
            a.record()
            fn()
            b.record()
            torch.cuda.synchronize()
            ms.append(a.elapsed_time(b))
        return sorted(ms)[len(ms) // 2]

    def one_at_a_time():
        seq.len = L
        for i in range(T):
            seq.append(k[i], v[i])
            seq.attend(q[i], rope_theta=theta)

    chunk_ms = timed(lambda: lc.attend_chunk(q, k, v, rope_theta=theta), 10)
    seq_ms = timed(one_at_a_time, 3)
    chunk = {"cache_tokens": L, "chunk_tokens": T, "shape": "llama7b_4bit", "attend_chunk_ms": chunk_ms,
             "append_plus_attend_loop_ms": seq_ms, "speedup": seq_ms / chunk_ms,
             "timing": "median of 10 (chunk) / 3 (per-token loop) runs, CUDA events, one layer"}

    line = {"what": "LayerCache.dequantize / attend_chunk, batch 1, one GPU", "gpu": gpu_info(0),
            "dequant": dequant,
            "dequant_timing": "median of %d single calls (CUDA events), alternating between 2 caches" % args.calls,
            "chunk": chunk, "peak_gbs": PEAK_GBS,
            "peak_source": "H100 SXM data sheet HBM3 bandwidth (3.35 TB/s), not a measured peak"}
    s = json.dumps(line)
    print(s, flush=True)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            f.write(s + "\n")
    return 0


if __name__ == "__main__":
    sys.exit(main())
