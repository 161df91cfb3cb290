#!/usr/bin/env python3
"""Length-dependent rotary frequencies (dynamic NTK, LongRoPE): what they cost on the GPU.  Prints one JSON line.

    python scripts/measure_rope_length.py [--iters N]

* kvq_rope_len_update (prepare + rebuild) of one sequence's state at 32K, 128K and 1M positions: when the frequencies
  do not change (below the switch: the rebuild exits at once) and when they change every step (dynamic NTK past the
  switch: positions [0, s) rewritten);
* the fused attend of one LLaMA-3-8B-shaped layer (32 query heads over 8 KV heads, 4 bits, K+V outliers, about 1 %
  each) at the same lengths, dynamic NTK (factor 4, max_position_embeddings 8192, its state prepared inside the call)
  against LLaMA-3.1's static llama3 frequencies;
* the 2-layer one-graph decode step (GraphedStage, dynamic) at 128K, dynamic NTK against llama31_8b(), alternated
  twice; the dynamic step's s changes every replay, so each replay rebuilds its table.
CUDA events around many launches after a warm-up; the card's name, power limit and SM clock are read in the same run.
"""
import argparse
import json
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
sys.path.insert(0, os.path.join(ROOT, "scripts"))
from measure_rope_scaling import gpu_info, time_us  # noqa: E402

DYN = dict(rope_type="dynamic", factor=4.0)


def spec():
    from kvquant_b200.rope import LengthDependentRotary
    return LengthDependentRotary(500000.0, DYN, 8192)


def update_times(iters):
    from kvquant_b200.cache import RopeLenState
    res = {}
    for L in (32768, 131072, 1 << 20):
        st = RopeLenState(spec(), 1, L + 1, "cuda:0")
        st.update(s=100)
        same = time_us(lambda: st.update(s=100), iters)
        flip = [L - 1]

        def changing():
            flip[0] = 2 * L - 1 - flip[0]                  # L - 1, L, L - 1, ...: a new key every call
            st.update(s=flip[0])
        res[str(L)] = {"unchanged_us": round(same, 2), "rebuild_us": round(time_us(changing, iters), 2)}
        del st
        torch.cuda.empty_cache()
    return res


def attend_times(iters):
    import test_gpu_gqa as G
    from kvquant_b200.rope import RotarySpec
    llama3 = RotarySpec(500000.0, {"rope_type": "llama3", "factor": 8.0, "low_freq_factor": 1.0,
                                   "high_freq_factor": 4.0, "original_max_position_embeddings": 8192})
    res = {}
    for L in (32768, 131072, 1 << 20):
        lc = G._cache(4, 32, 8, "kv", Lmax=L + 4)
        k, v = G._tokens(lc, 8192, seed=1)
        for _ in range(0, L, 8192):
            lc.append_chunk(k, v)
        q = G._query(32, 1)
        out = torch.empty((32, 128), device="cuda:0")
        row = {}
        for rep in range(2):                               # alternated: spread is the difference of the repeats
            for name, r in (("llama3", llama3), ("dynamic", spec())):
                row.setdefault(name + "_attend_us", []).append(
                    round(time_us(lambda: lc.attend(q, rope=r, out=out), iters), 2))
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
    stages = {}
    for name, cfg in (("llama31_8b", kd.DecodeConfig.llama31_8b(n_layers=2, max_len=L + 64)),
                      ("dynamic", kd.DecodeConfig.llama3_8b(n_layers=2, max_len=L + 64, rope_scaling=DYN,
                                                            max_position_embeddings=8192))):
        st = kd.DecoderStage(cfg, 0, 2, "cuda:0", quant, seed=1, with_head=True)
        g = torch.Generator(device="cuda:0").manual_seed(0)
        for ly in st.layers:
            k = torch.randn((8192, cfg.kv_hidden), generator=g, device="cuda:0")
            v = torch.randn((8192, cfg.kv_hidden), generator=g, device="cuda:0")
            for _ in range(L // 8192):
                ly.cache.append_chunk(k, v)
        stages[name] = (st, kd.GraphedStage(st, L, first=True, last_to_logits=True, dynamic=True))
    res = {}
    for rep in range(2):
        for name, (st, gs) in stages.items():
            flip = [L - 1]

            def step():
                flip[0] = 2 * L - 1 - flip[0]
                st.set_device_length(flip[0], flip[0])
                gs.graph.replay()
            res.setdefault(name + "_step_us_2layers", []).append(round(time_us(step, iters), 2))
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=50)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("needs a CUDA device")
    out = {"gpu": gpu_info(), "rope_len_update": update_times(a.iters),
           "attend_layer_llama3_8b_4bit": attend_times(a.iters), "decode_128k": decode_step(a.iters)}
    print(json.dumps(out))


if __name__ == "__main__":
    main()
