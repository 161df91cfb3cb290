#!/usr/bin/env python
"""Two-KV-head and multi-query models over the quantised cache: the per-layer fused decode attend at H_kv = 2 and 1
against kvq_attend over the same cache replicated into one KV head per query head (synth.replicate_kv_heads), and a
one-graph 36-layer decode step of the Qwen2.5-3B attention shape (16 query heads over 2 KV heads, hidden 2048).

    python scripts/measure_small_kv.py [--lengths 32768 131072 1048576] [--calls 50] [--steps 20] [--out FILE]

Prints one JSON line:
  * gpu: card name, power limit and maximum SM clock, read in the same run;
  * attend: per shape (16/2 and 32/2 at 4 and 3 bits, 32/1 at 4 bits; 1 % K and V outliers) and cache length, the
    median of `--calls` CUDA-event timings of each form, the two forms alternating call by call and each cycling over
    enough layers' caches to exceed the 50 MB L2; the bytes one call must read (LayerCache.bytes_per_token) of each
    form and the GQA form's GB/s from its own bytes;
  * decode: ms/step of the one-graph dynamic-length decode step of 36 layers of 16/2 (hidden 2048, intermediate
    11008, 4-bit + 1 %) at the first length >= 128K (default 128K), median over `--steps` replays after 3 warm-ups.
"""
import argparse
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "scripts"))

from measure_dequant import CACHE_TENSORS  # noqa: E402
from measure_gqa import L2_BYTES, alternate, gqa_caches, quantizer  # noqa: E402
from measure_wide_heads import gpu_info  # noqa: E402

SHAPES = ((16, 2, 4), (16, 2, 3), (32, 2, 4), (32, 2, 3), (32, 1, 4))


def attend_rows(lengths, calls, dev):
    import torch
    from kvquant_b200 import synth
    rows = []
    for Hq, Hkv, bits in SHAPES:
        for L in lengths:
            b_gqa = gqa_caches(Hq, Hkv, bits, 32, 1, dev)[0].bytes_per_token() * L
            n = max(2, -(-2 * L2_BYTES // b_gqa))
            caches = gqa_caches(Hq, Hkv, bits, L, n, dev)
            mha = [synth.replicate_kv_heads(c) for c in caches[:2]]   # (the replicas alone exceed L2)
            q = torch.randn((Hq, 128), device=dev).half().float()
            outs = [torch.empty((Hq, 128), device=dev) for _ in range(2)]
            g_ms, m_ms = alternate([[lambda c=c: c.attend(q, out=outs[0]) for c in caches],
                                    [lambda c=c: c.attend(q, out=outs[1]) for c in mha]], calls)
            diff = ((outs[0] - outs[1]).norm() / outs[1].norm()).item()
            rows.append(dict(q_heads=Hq, kv_heads=Hkv, bits=bits, tokens=L, caches=n, gqa_ms=g_ms,
                             replicated_mha_ms=m_ms, gqa_bytes_per_token=b_gqa // L,
                             replicated_bytes_per_token=mha[0].bytes_per_token(), gqa_gbs=b_gqa / g_ms / 1e6,
                             rel_diff=diff))
            print(json.dumps(rows[-1]), file=sys.stderr, flush=True)
            del caches, mha
            torch.cuda.empty_cache()
    return rows


def decode_row(L, steps, dev):
    import torch
    from kvquant_b200 import decode as kd, synth
    cfg = kd.DecodeConfig(n_layers=36, hidden=2048, n_heads=16, n_kv_heads=2, intermediate=11008, vocab=32000,
                          rope_theta=1e6, bits=4, max_len=L + steps + 16)
    sp, qz = quantizer(cfg.kv_heads, 4, dev)
    st = kd.DecoderStage(cfg, 0, cfg.n_layers, dev, qz, seed=0, with_head=True)
    first = st.layers[0].cache
    synth.fill_layer_cache_gpu(first, sp, L, seed=0)
    for ly in st.layers[1:]:
        for name in CACHE_TENSORS:
            getattr(ly.cache, name).copy_(getattr(first, name))
        ly.cache.len = L
    gs = kd.GraphedStage(st, L, first=True, last_to_logits=True, dynamic=True)
    gs.tok.fill_(1)
    for _ in range(3):
        gs.replay()
    torch.cuda.synchronize()
    ev = [(torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)) for _ in range(steps)]
    for a, b in ev:
        a.record()
        gs.replay()
        b.record()
    torch.cuda.synchronize()
    ms = sorted(a.elapsed_time(b) for a, b in ev)[steps // 2]
    ok = bool(torch.isfinite(gs.logits.float()).all().item())
    row = dict(q_heads=16, kv_heads=2, hidden=2048, layers=cfg.n_layers, bits=4, tokens=L, ms_per_step=ms,
               finite_logits=ok, cache_bytes_per_step=cfg.n_layers * kd.layer_step_bytes(cfg, L))
    del gs, st
    torch.cuda.empty_cache()
    return row


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--lengths", type=int, nargs="+", default=[32768, 131072, 1048576])
    ap.add_argument("--calls", type=int, default=50)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--out", default=None, help="also write the JSON line to this file")
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("measure_small_kv.py needs a CUDA device")
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    res = dict(gpu=gpu_info(0), attend=attend_rows(args.lengths, args.calls, dev))
    res["decode"] = decode_row(min([x for x in args.lengths if x >= 131072] or [max(args.lengths)]), args.steps, dev)
    line = json.dumps(res)
    print(line)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
