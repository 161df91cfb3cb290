#!/usr/bin/env python3
"""Scaled rotary frequencies: what they cost on the GPU.  Prints one JSON line.

    python scripts/measure_rope_scaling.py [--iters N]

* the fused attend of one LLaMA-3-8B-shaped layer (32 query heads over 8 KV heads, 4 bits, K+V outliers) at 32K, 128K
  and 1M cached tokens, with rope_theta = 500000 against LLaMA-3.1's llama3 frequencies against linear x8; the K outlier
  pass alone is the attend with the outlier rows against the same attend with K outliers only in V (reported as the
  difference of the two);
* the 2-layer one-graph decode step (GraphedStage, dynamic) of llama31_8b() against llama3_8b() at 128K, scaled to 32
  layers by the layer count.
CUDA events around many launches after a warm-up; the card's name, power limit and SM clock are read in the same run.
"""
import argparse
import json
import os
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))


def gpu_info():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm,clocks.sm",
                              "--format=csv,noheader"], capture_output=True, text=True, timeout=30).stdout.strip()
    except OSError:
        out = ""
    return out.splitlines()[0] if out else torch.cuda.get_device_name(0)


def time_us(fn, iters):
    for _ in range(3):
        fn()
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(iters):
        fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) * 1e3 / iters


def attend_times(iters):
    import test_gpu_gqa as G
    from kvquant_b200.rope import RotarySpec
    specs = {"theta": None,
             "llama3": RotarySpec(500000.0, {"rope_type": "llama3", "factor": 8.0, "low_freq_factor": 1.0,
                                             "high_freq_factor": 4.0, "original_max_position_embeddings": 8192}),
             "linear": RotarySpec(500000.0, {"rope_type": "linear", "factor": 8.0})}
    res = {}
    for L in (32768, 131072, 1 << 20):
        lc = G._cache(4, 32, 8, "kv", Lmax=L + 4)
        k, v = G._tokens(lc, 8192, seed=1)
        for s0 in range(0, L, 8192):
            lc.append_chunk(k, v)
        q = G._query(32, 1)
        out = torch.empty((32, 128), device="cuda:0")
        row = {}
        for name, spec in specs.items():
            row[name + "_attend_us"] = round(time_us(lambda: lc.attend(q, rope_theta=500000.0, rope=spec, out=out),
                                                     iters), 2)
        lc.sparse_k = False          # the same attend without the K outlier pass
        for name, spec in specs.items():
            t = time_us(lambda: lc.attend(q, rope_theta=500000.0, rope=spec, out=out), iters)
            row[name + "_kout_us"] = round(row[name + "_attend_us"] - t, 2)
        lc.sparse_k = True
        res[str(L)] = row
        del lc
        torch.cuda.empty_cache()
    return res


def decode_step(iters):
    from kvquant_b200 import cache as kc, decode as kd, synth
    sp = synth.SynthSpec(8, 128, seed=0)
    cal = synth.calibrate(sp, 4, calib_tokens=256, seed=7)
    t = kc.build_k_lookup_table(cal["k"][0], cal["k"][1], cal["k"][2][0], 8, device="cuda:0")
    quant = dict(klut=dict(lut=t["lut"], lut2=None, thr_lower=t["thr_lower"], thr_upper=t["thr_upper"]),
                 v_cent=cal["v"][2][0])
    L = 131072
    res = {}
    for name, mk in (("llama3_8b", kd.DecodeConfig.llama3_8b), ("llama31_8b", kd.DecodeConfig.llama31_8b)):
        cfg = mk(n_layers=2, max_len=L + 64)
        st = kd.DecoderStage(cfg, 0, 2, "cuda:0", quant, seed=1, with_head=True)
        g = torch.Generator(device="cuda:0").manual_seed(0)
        for ly in st.layers:       # 128K synthetic pre-RoPE tokens per layer
            k = torch.randn((8192, cfg.kv_hidden), generator=g, device="cuda:0")
            v = torch.randn((8192, cfg.kv_hidden), generator=g, device="cuda:0")
            for _ in range(L // 8192):
                ly.cache.append_chunk(k, v)
        gs = kd.GraphedStage(st, L, first=True, last_to_logits=True, dynamic=True)

        def step():
            st.set_device_length(L, st.layers[0].cache.n_sink + L)
            gs.graph.replay()
        res[name + "_step_us_2layers"] = round(time_us(step, iters), 2)
        del gs, st
        torch.cuda.empty_cache()
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=50)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("needs a CUDA device")
    from kvquant_b200 import build
    build.build(verbose=False)
    out = {"gpu": gpu_info(), "attend_layer_llama3_8b_4bit": attend_times(a.iters), "decode_128k": decode_step(a.iters)}
    print(json.dumps(out))


if __name__ == "__main__":
    main()
