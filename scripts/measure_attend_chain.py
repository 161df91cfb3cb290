#!/usr/bin/env python
"""Where one decode step's time goes: per-kernel device times of one layer's fused attend, and the idle time between
the kernels of a whole step (DESIGN.md section 5).

    python scripts/measure_attend_chain.py --out DIR [--workload 7b-3b-128k] [--steps 3] [--warmup 3]

Builds the workload's decoder stage and one-graph dynamic decode step as bench.py does, replays it `--warmup` times,
then records `--steps` replays under torch.profiler (CUDA activities only) in a run of its own and writes:
  * DIR/attend_chain.pt.trace.json: the raw trace;
  * DIR/attend_chain.md: the tables below;
and prints one JSON line with:
  * gpu: card name, power limit and maximum SM clock, read in the same run;
  * attend: per launch of one layer's attend chain (attend_init .. attend_combine), the median over all layers and
    steps of its device time and of the gap since the previous launch ended (negative: the two overlapped);
  * step: per replay, the span from the first launch's start to the last launch's end, the summed device time, the
    idle time (sum of the positive gaps) and the launch count; and the step's kernels by total time.
"""
import argparse
import json
import os
import re
import sys
from collections import defaultdict

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "scripts"))

import bench  # noqa: E402
from measure_wide_heads import gpu_info  # noqa: E402

DEVICE_CATS = ("kernel", "gpu_memset", "gpu_memcpy")


def short_name(name):
    """Kernel name without namespace, return type, argument list or template arguments past the first."""
    n = re.sub(r"^void\s+", "", name)
    n = n.split("(")[0]
    n = n.replace("kvq::", "")
    m = re.match(r"([^<]+)(<[^,>]*)?", n)
    return (m.group(1) + ((m.group(2) + ",..>") if m.group(2) else "")) if m else n


def median(xs):
    s = sorted(xs)
    return s[len(s) // 2] if s else None


def device_events(trace_path):
    with open(trace_path) as f:
        tr = json.load(f)
    evs = [e for e in tr.get("traceEvents", []) if e.get("ph") == "X" and e.get("cat") in DEVICE_CATS]
    evs.sort(key=lambda e: e["ts"])
    return [(short_name(e["name"]) if e["cat"] == "kernel" else e["cat"], float(e["ts"]), float(e["dur"])) for e in evs]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", required=True, help="output directory (trace and tables)")
    ap.add_argument("--workload", default=bench.DEFAULT_WORKLOAD, choices=sorted(bench.WORKLOADS))
    ap.add_argument("--steps", type=int, default=3)
    ap.add_argument("--warmup", type=int, default=3)
    args = ap.parse_args()

    import torch
    from torch.profiler import ProfilerActivity, profile
    from kvquant_b200 import decode as kd, synth

    os.makedirs(args.out, exist_ok=True)
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    gpu = gpu_info(0)
    model, bits, L, n_sink, outl, _ = bench.WORKLOADS[args.workload]
    headroom = (2 * (args.steps + args.warmup) + 3 + 8 + 63) // 64 * 64
    mk = kd.DecodeConfig.llama13b if model == "13b" else kd.DecodeConfig.llama7b
    cfg = mk(bits=bits, n_sink=n_sink, max_len=L + headroom, include_sparse=(outl != "none"), sparse_v=(outl == "kv"))
    sp, quantizer = bench.build_quantizer(bits, cfg.n_heads, dev)
    stage = kd.DecoderStage(cfg, 0, cfg.n_layers, dev, quantizer, seed=0, with_head=True)
    for i, ly in enumerate(stage.layers):
        synth.fill_layer_cache_gpu(ly.cache, sp, L, seed=i * 16)
    torch.cuda.synchronize()
    gs = kd.GraphedStage(stage, L, first=True, last_to_logits=True, dynamic=True)
    for _ in range(args.warmup):
        gs.replay()
    torch.cuda.synchronize()

    trace = os.path.join(args.out, "attend_chain.pt.trace.json")
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(args.steps):
            gs.replay()
            torch.cuda.synchronize()
    prof.export_chrome_trace(trace)

    evs = device_events(trace)
    if len(evs) % args.steps:
        raise SystemExit("%d device events are not %d equal steps" % (len(evs), args.steps))
    per = len(evs) // args.steps
    steps, attend_rows, totals = [], defaultdict(list), defaultdict(float)
    for s in range(args.steps):
        ev = evs[s * per:(s + 1) * per]
        gaps = [ev[i][1] - (ev[i - 1][1] + ev[i - 1][2]) for i in range(1, len(ev))]
        steps.append({"span_us": ev[-1][1] + ev[-1][2] - ev[0][1], "busy_us": sum(e[2] for e in ev),
                      "idle_us": sum(g for g in gaps if g > 0), "overlap_us": -sum(g for g in gaps if g < 0),
                      "launches": len(ev)})
        for name, _, dur in ev:
            totals[name] += dur / args.steps
        i = 0
        while i < len(ev):       # every layer's attend chain: attend_init .. attend_combine
            if ev[i][0].startswith("attend_init"):
                j = i
                while j < len(ev) and not ev[j][0].startswith("attend_combine"):
                    j += 1
                for k in range(i, min(j + 1, len(ev))):
                    attend_rows[k - i].append((ev[k][0], ev[k][2], ev[k][1] - (ev[k - 1][1] + ev[k - 1][2])))
                i = j
            i += 1
    attend = [{"kernel": rows[0][0], "us": median([r[1] for r in rows]), "gap_before_us": median([r[2] for r in rows]),
               "samples": len(rows)} for _, rows in sorted(attend_rows.items())]
    top = sorted(totals.items(), key=lambda kv: -kv[1])[:16]
    res = {"workload": args.workload, "gpu": gpu, "steps": steps,
           "attend": attend, "attend_sum_us": sum(a["us"] for a in attend),
           "step_kernels_us": [{"kernel": k, "us_per_step": v} for k, v in top]}

    with open(os.path.join(args.out, "attend_chain.md"), "w") as f:
        f.write("%s, %s, power limit %s W\n\n" % (args.workload, gpu["name"], gpu["power_limit_w"]))
        f.write("| # | kernel (one layer's attend) | us | gap before, us |\n|---|---|---|---|\n")
        for i, a in enumerate(attend):
            f.write("| %d | %s | %.1f | %.1f |\n" % (i, a["kernel"], a["us"], a["gap_before_us"]))
        f.write("\n| step | span, us | busy, us | idle, us | overlap, us | launches |\n|---|---|---|---|---|---|\n")
        for i, s in enumerate(steps):
            f.write("| %d | %.0f | %.0f | %.0f | %.0f | %d |\n" % (i, s["span_us"], s["busy_us"], s["idle_us"],
                                                                s["overlap_us"], s["launches"]))
        f.write("\n| kernel | us per step |\n|---|---|\n")
        for k, v in top:
            f.write("| %s | %.0f |\n" % (k, v))
    print(json.dumps(res), flush=True)
    return 0


if __name__ == "__main__":
    sys.exit(main())
