#!/usr/bin/env python
"""LLaMA-13B at 4 bits + 1 % outliers on one GPU: the shape whose native V pass runs in two head groups.

    python scripts/measure_wide_heads.py [--lengths 32768 131072] [--calls 200] [--steps 20] [--warmup 3]

Prints one JSON line:
  * gpu: card name, power limit and maximum SM clock, read in the same run;
  * attend: per-layer fused-attend time at each length, for the native form (head-split V pass) and for the
    per-token-LUT form (LayerCache.use_native_v = False).  Median of `--calls` calls timed one by one with CUDA events
    after a warm-up, cycling over all 40 layers' caches so that L2 (50 MB) cannot serve a cache (6016 B/token x 32K
    tokens is already 197 MB).  Exact fp32 K tables in both forms.  GB/s are algorithmic bytes (SURVEY.md 8d:
    2*hidden*bits/8 + 4*2^bits + 2*n_out*8 per token) over the median time, and their fraction of the H100 SXM data
    sheet's 3.35 TB/s;
  * decode: tokens/s of the one-graph decode loop (device-resident length, every replay is the next step of a growing
    cache) for the whole 40-layer model at the largest length.

Weights are random-init fp16.  Layer 0's cache is filled with synthetic K/V through the real prefill packers and
copied to the other layers (distinct memory, same contents: the timing depends on the bytes streamed, not on them).
Needs about 26 GB of weights plus 6016 B x 40 layers per token of cache (31.5 GB at 128K): one 80 GB GPU.
"""
import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

PEAK_GBS = 3350.0   # H100 SXM data sheet HBM3 bandwidth, not a measured peak
CACHE_TENSORS = ("kcache", "vcache", "vlut", "vaff", "k_outliers", "k_outlier_idx", "v_outliers", "v_outlier_idx")


def gpu_info(index):
    import torch
    info = {"name": torch.cuda.get_device_name(index), "power_limit_w": None, "sm_max_mhz": None}
    try:
        out = subprocess.run(["nvidia-smi", "-i", str(index), "--query-gpu=power.limit,clocks.max.sm",
                              "--format=csv,noheader,nounits"], capture_output=True, text=True, timeout=30).stdout
        f = [x.strip() for x in out.strip().split(",")]
        info["power_limit_w"], info["sm_max_mhz"] = float(f[0]), float(f[1])
    except Exception as e:  # noqa: BLE001  (reported as missing, never guessed)
        info["error"] = repr(e)[:120]
    return info


def median_call_ms(fn, caches, calls, warm):
    """Median over `calls` single calls, each bracketed by its own pair of CUDA events, cycling over `caches`."""
    import torch
    for i in range(warm):
        fn(caches[i % len(caches)])
    torch.cuda.synchronize()
    ev = [(torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)) for _ in range(calls)]
    for i, (a, b) in enumerate(ev):
        a.record()
        fn(caches[i % len(caches)])
        b.record()
    torch.cuda.synchronize()
    ms = sorted(a.elapsed_time(b) for a, b in ev)
    return ms[len(ms) // 2]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--lengths", type=int, nargs="+", default=[32768, 131072])
    ap.add_argument("--calls", type=int, default=200)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    args = ap.parse_args()
    if args.calls < 100:
        raise SystemExit("--calls must be at least 100")

    import torch
    from kvquant_b200 import decode as kd, synth, cache as kc
    if not torch.cuda.is_available():
        raise SystemExit("needs a CUDA device")
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    L = max(args.lengths)
    bits = 4
    headroom = (args.steps + 2 * args.warmup + 8 + 63) // 64 * 64
    cfg = kd.DecodeConfig.llama13b(bits=bits, max_len=L + headroom)
    H = cfg.n_heads
    sp = synth.SynthSpec(H, 128, seed=0)
    cal = synth.calibrate(sp, bits, calib_tokens=512, seed=7)
    t = kc.build_k_lookup_table(cal["k"][0], cal["k"][1], cal["k"][2][0], H, device=dev)
    quant = dict(klut=dict(lut=t["lut"], lut2=None, thr_lower=t["thr_lower"], thr_upper=t["thr_upper"]),
                 v_cent=cal["v"][2][0])
    stage = kd.DecoderStage(cfg, 0, cfg.n_layers, dev, quant, seed=0, with_head=True)
    caches = [ly.cache for ly in stage.layers]
    synth.fill_layer_cache_gpu(caches[0], sp, L, seed=0)
    for lc in caches[1:]:
        for name in CACHE_TENSORS:
            getattr(lc, name).copy_(getattr(caches[0], name))
        lc.len = caches[0].len
    torch.cuda.synchronize()
    per_tok = caches[0].bytes_per_token()

    # ---- per-layer fused attend: native (head-split V pass) vs per-token-LUT V pass ----------------------------
    q = torch.randn((H, 128), generator=torch.Generator(device=dev).manual_seed(5), device=dev).half().float()
    attend = []
    for Lt in sorted(args.lengths):
        for lc in caches:
            lc.len = Lt
        rec = {"tokens": Lt, "bytes": Lt * per_tok}
        outs = {}
        for form, native in (("native_split", True), ("per_token_lut", False)):
            for lc in caches:
                lc.use_native_v = native
                lc.precision = "fp32"
            ms = median_call_ms(lambda lc: lc.attend(q, rope_theta=cfg.rope_theta), caches, args.calls, warm=2 * len(caches))
            gbs = Lt * per_tok / ms / 1e6
            rec[form] = {"ms": ms, "gbs": gbs, "frac_of_3350": gbs / PEAK_GBS}
            outs[form] = caches[0].attend(q, rope_theta=cfg.rope_theta).clone()
        rec["lut_over_native_time"] = rec["per_token_lut"]["ms"] / rec["native_split"]["ms"]
        rec["native_vs_lut_rel_diff"] = ((outs["native_split"] - outs["per_token_lut"]).abs().max()
                                         / outs["per_token_lut"].abs().max()).item()
        attend.append(rec)
    for lc in caches:
        lc.use_native_v = True
        lc.len = L

    # ---- whole-model one-graph decode loop at L ----------------------------------------------------------------
    gs = kd.GraphedStage(stage, L, first=True, last_to_logits=True, dynamic=True)
    for _ in range(args.warmup):
        gs.replay()
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(args.steps):
        gs.replay()
    b.record()
    torch.cuda.synchronize()
    ms_step = a.elapsed_time(b) / args.steps
    logits_ok = bool(torch.isfinite(gs.logits.float()).all().item())

    line = {
        "what": "LLaMA-13B 4-bit NUQ + 1% outliers (K and V), batch 1, one GPU",
        "gpu": gpu_info(0),
        "bytes_per_token_per_layer": per_tok,
        "attend_per_layer": attend,
        "attend_timing": "median of %d single calls (CUDA events), cycling over %d layers' caches, exact fp32 K tables"
                         % (args.calls, len(caches)),
        "decode": {"tokens": L, "layers": cfg.n_layers, "steps": args.steps, "warmup": args.warmup,
                   "ms_per_step": ms_step, "tokens_per_s": 1000.0 / ms_step, "logits_finite": logits_ok,
                   "weight_bytes": stage.weight_bytes(), "cache_bytes_per_step": cfg.n_layers * L * per_tok},
        "peak_gbs": PEAK_GBS,
        "peak_source": "H100 SXM data sheet HBM3 bandwidth (3.35 TB/s), not a measured peak",
    }
    print(json.dumps(line), flush=True)
    return 0


if __name__ == "__main__":
    sys.exit(main())
