#!/usr/bin/env python
"""Device time of the K-outlier pass (`k_outlier_pers_kernel`) of one layer's fused attend, per build and cache length
(DESIGN.md section 5).

    python scripts/measure_kout.py --arm new=kvquant_b200/libkvquant_b200.so --arm old=OTHER.so[,ENV=VALUE...]
                                   [--lengths 32768 131072 1048576] [--bits 3] [--rounds 3] [--calls 60]

Each arm is a name, a built libkvquant_b200.so and optional environment settings (for example
KVQ_KOUT_DIRECT_NPOS=1000000000 to force the rope-table gather).  The arms run one after another in fresh processes,
`--rounds` times in turn, so that two builds are compared alternately in one session.  A process loads its arm's
library, fills one LLaMA-7B-shaped layer cache (32 heads, 1 % K and V outliers; the first 128K tokens are synthetic
K/V through the real packers, longer caches repeat them), and for each length records `--calls` fused attends under
torch.profiler (CUDA activities only).  Prints one JSON line with the card name and power limit read in the same run
and, per length and arm, the median outlier-pass time over all calls and the median of each round.
"""
import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "scripts"))

KERNEL = "k_outlier_pers_kernel"
FILL_TOKENS = 131072


def median(xs):
    s = sorted(xs)
    return s[len(s) // 2] if s else None


def child(args):
    from kvquant_b200 import _lib
    _lib.LIB_PATH = os.path.abspath(args.lib)
    import torch
    from torch.profiler import ProfilerActivity, profile
    import bench
    from kvquant_b200 import cache as kc, synth
    from measure_wide_heads import gpu_info

    if not torch.cuda.is_available():
        raise SystemExit("needs a CUDA device")
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    H, Lmax = 32, max(args.lengths)
    sp, qz = bench.build_quantizer(args.bits, H, dev)
    lc = kc.LayerCache.from_luts(args.bits, H, Lmax + 64, qz["klut"], qz["v_cent"], device=dev)
    n = min(Lmax, FILL_TOKENS)
    synth.fill_layer_cache_gpu(lc, sp, n, seed=0, chunk=16384)
    tok_major = ("k_outliers", "k_outlier_idx", "v_outliers", "v_outlier_idx", "vlut", "vaff")
    for t0 in range(n, Lmax, n):
        t1 = min(Lmax, t0 + n)
        for name in ("kcache", "vcache"):
            x = getattr(lc, name)
            x[:, :, t0:t1] = x[:, :, :t1 - t0]
        for name in tok_major:
            x = getattr(lc, name)
            x[t0:t1] = x[:t1 - t0]
    q = torch.randn((H, 128), generator=torch.Generator(device=dev).manual_seed(5), device=dev).half().float()
    res = {"gpu": gpu_info(0), "us": {}}
    for L in args.lengths:
        lc.len = L
        for _ in range(5):
            lc.attend(q)
        torch.cuda.synchronize()
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            for _ in range(args.calls):
                lc.attend(q)
            torch.cuda.synchronize()
        us = [e.device_time for e in prof.events() if KERNEL in e.name and e.device_time > 0]
        if len(us) != args.calls:
            raise SystemExit("%d %s launches recorded for %d calls" % (len(us), KERNEL, args.calls))
        res["us"][str(L)] = us
    print("RESULT " + json.dumps(res), flush=True)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--arm", action="append", default=[], help="NAME=LIB[,ENV=VALUE...]")
    ap.add_argument("--lengths", type=int, nargs="+", default=[32768, 131072, 1048576])
    ap.add_argument("--bits", type=int, default=3, choices=(2, 3, 4))
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--calls", type=int, default=60)
    ap.add_argument("--child", action="store_true", help=argparse.SUPPRESS)
    ap.add_argument("--lib", default="", help=argparse.SUPPRESS)
    args = ap.parse_args()
    if args.child:
        return child(args)
    if not args.arm:
        raise SystemExit("give at least one --arm NAME=LIB")
    arms = []
    for spec in args.arm:
        name, rest = spec.split("=", 1)
        parts = rest.split(",")
        env = dict(p.split("=", 1) for p in parts[1:])
        arms.append((name, parts[0], env))
    samples = {str(L): {a[0]: [] for a in arms} for L in args.lengths}
    rounds = {str(L): {a[0]: [] for a in arms} for L in args.lengths}
    gpu = None
    for _ in range(args.rounds):
        for name, lib, env in arms:
            cmd = [sys.executable, os.path.abspath(__file__), "--child", "--lib", lib, "--bits", str(args.bits),
                   "--calls", str(args.calls), "--lengths"] + [str(L) for L in args.lengths]
            out = subprocess.run(cmd, env=dict(os.environ, **env), capture_output=True, text=True)
            line = [x for x in out.stdout.splitlines() if x.startswith("RESULT ")]
            if out.returncode != 0 or not line:
                sys.stderr.write(out.stdout[-2000:] + out.stderr[-4000:])
                raise SystemExit("arm %s failed (exit %d)" % (name, out.returncode))
            r = json.loads(line[0][len("RESULT "):])
            gpu = gpu or r["gpu"]
            for L, us in r["us"].items():
                samples[L][name] += us
                rounds[L][name].append(median(us))
    table = {L: {name: {"median_us": median(samples[L][name]), "round_medians_us": rounds[L][name],
                        "calls": len(samples[L][name])} for name, _, _ in arms} for L in samples}
    print(json.dumps({"kernel": KERNEL, "gpu": gpu, "bits": args.bits, "heads": 32,
                      "arms": {name: {"lib": lib, "env": env} for name, lib, env in arms}, "per_layer": table}),
          flush=True)
    return 0


if __name__ == "__main__":
    sys.exit(main())
