#!/usr/bin/env python
"""Ragged prefill (DESIGN.md section 4.15): BatchedDecoderStage.prefill_seqs against the loop of prefill_seq, and the
ragged append / attend of one layer against the per-slot calls.

    python scripts/measure_ragged_prefill.py [--layers 32] [--reps 2] [--page 640] [--models llama3_8b,llama7b]

Prints one JSON line:
  * gpu: card name, power limit and maximum SM clock, read in the same run;
  * grid_<model>: per model (LLaMA-3-8B 32/8 and LLaMA-7B 32/32 shapes, 4-bit, 1 % K and V outliers, `--layers` layers) and
    cache kind (paged with `--page`-token pages, contiguous): k in (4, 16, 64) prompts of T in (128, 512, 2048) tokens
    into empty slots, prefill_seqs (chunk 2048, max_tokens 8192) against prefill_seq of each prompt in turn, alternating
    over `--reps` repetitions; median wall-clock seconds to the last commit (synchronised) and prompt tokens/s;
  * fork: 16 forks of a 4096-token prefix (paged), each given a 256-token suffix: prefill_seqs of the 16 suffixes
    against the prefill_seq loop (the forks are rebuilt between repetitions);
  * follow_up: one 512-token follow-up into a slot holding 32768 tokens (paged; length restored between repetitions):
    prefill_seqs({b: y}) against prefill_seq(b, y).  The fused chunk attend reads the whole 32K-token slot per chunk,
    the SDPA route dequantises it once: this is the case where the fused kernel is known to lose (section 4.8);
  * kernels: one LLaMA-3-8B-shaped layer, 16 slots of 512 tokens each holding 512 tokens already: CUDA-event ms of one
    append_chunks against 16 append_chunk calls, and of one attend_chunks against 16 attend_chunk_fused calls
    (contiguous), and of the paged append forms.
"""
import argparse
import json
import os
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "scripts"))

from measure_wide_heads import gpu_info  # noqa: E402
from measure_paged_prefill import calibration  # noqa: E402

THETA = 10000.0


def seconds(fn):
    import torch
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    fn()
    torch.cuda.synchronize()
    return time.perf_counter() - t0


def med(t):
    return sorted(t)[len(t) // 2]


def make_stage(model, layers, max_len, dev):
    from kvquant_b200 import decode as kd
    if model == "llama3_8b":
        cfg = kd.DecodeConfig.llama3_8b(n_layers=layers, bits=4, max_len=max_len)
    else:
        cfg = kd.DecodeConfig(n_layers=layers, hidden=4096, n_heads=32, intermediate=11008, vocab=32000, bits=4,
                              max_len=max_len)
    klut, vcent, _, _ = calibration(cfg.kv_heads, 4, dev)
    return kd.DecoderStage(cfg, 0, layers, dev, dict(klut=klut, v_cent=vcent), seed=1, with_head=True)


def prompts(st, k, T, seed, dev):
    import torch
    g = torch.Generator(device=dev).manual_seed(seed)
    return {b: st.embed[torch.randint(0, st.cfg.vocab, (T,), generator=g, device=dev)] for b in range(k)}


def race(loop, ragged, reps):
    """Median seconds of the two routes, alternating, after one warm-up of each."""
    loop(), ragged()
    t_l, t_r = [], []
    for _ in range(reps):
        t_l.append(seconds(loop))
        t_r.append(seconds(ragged))
    return med(t_l), med(t_r)


def measure_grid(model, layers, P, reps, dev):
    from kvquant_b200 import decode as kd
    st = make_stage(model, layers, 2048, dev)
    rows = []
    for paged in (True, False):
        for T in (128, 512, 2048):
            for k in (4, 16, 64):
                bst = kd.BatchedDecoderStage(st, k, page_size=P if paged else None)
                xs = prompts(st, k, T, k + T, dev)

                def loop():
                    for b in xs:
                        bst.reset_seq(b)
                    for b, x in xs.items():
                        bst.prefill_seq(b, x)

                def ragged():
                    for b in xs:
                        bst.reset_seq(b)
                    bst.prefill_seqs(xs)
                s_l, s_r = race(loop, ragged, reps)
                rows.append(dict(model=model, layers=layers, kind="paged" if paged else "contiguous", k=k, T=T,
                                 loop_s=round(s_l, 4), ragged_s=round(s_r, 4), loop_tok_s=round(k * T / s_l),
                                 ragged_tok_s=round(k * T / s_r), speedup=round(s_l / s_r, 3)))
                del bst
    return rows


def measure_fork(layers, P, reps, dev, prefix=4096, suffix=256, n=16):
    import torch
    from kvquant_b200 import decode as kd
    st = make_stage("llama3_8b", layers, prefix + suffix + 64, dev)
    bst = kd.BatchedDecoderStage(st, n + 1, page_size=P)
    g = torch.Generator(device=dev).manual_seed(3)
    bst.prefill_seq(0, st.embed[torch.randint(0, st.cfg.vocab, (prefix,), generator=g, device=dev)])
    xs = {b: x for b, x in prompts(st, n + 1, suffix, 4, dev).items() if b > 0}

    def refork():
        for b in xs:
            bst.reset_seq(b)
            bst.fork_seq(0, b)

    def loop():
        refork()
        for b, x in xs.items():
            bst.prefill_seq(b, x)

    def ragged():
        refork()
        bst.prefill_seqs(xs)
    s_l, s_r = race(loop, ragged, reps)
    return dict(model="llama3_8b", layers=layers, prefix=prefix, forks=n, suffix=suffix, loop_s=round(s_l, 4),
                ragged_s=round(s_r, 4), speedup=round(s_l / s_r, 3), note="timings include the forks' page copies")


def measure_follow_up(layers, P, reps, dev, held=32768, follow=512):
    import torch
    from kvquant_b200 import decode as kd
    st = make_stage("llama3_8b", layers, held + follow + 64, dev)
    bst = kd.BatchedDecoderStage(st, 1, page_size=P)
    g = torch.Generator(device=dev).manual_seed(5)
    bst.prefill_seq(0, st.embed[torch.randint(0, st.cfg.vocab, (held,), generator=g, device=dev)])
    y = st.embed[torch.randint(0, st.cfg.vocab, (follow,), generator=g, device=dev)]

    def restore():
        bst.pages.lens_host[0] = held
        bst.caches[0].commit(0)

    def loop():
        restore()
        bst.prefill_seq(0, y)

    def ragged():
        restore()
        bst.prefill_seqs({0: y})
    s_l, s_r = race(loop, ragged, reps)
    return dict(model="llama3_8b", layers=layers, held=held, T=follow, loop_s=round(s_l, 4), ragged_s=round(s_r, 4),
                speedup=round(s_l / s_r, 3))


def events(fn, calls):
    import torch
    fn()
    ts = []
    for _ in range(calls):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        fn()
        b.record()
        torch.cuda.synchronize()
        ts.append(a.elapsed_time(b))
    return med(ts)


def measure_kernels(P, calls, dev, k=16, T=512, L=512):
    import torch
    from kvquant_b200 import cache as kc
    Hq, Hkv = 32, 8
    klut, vcent, mu, sigma = calibration(Hkv, 4, dev)
    bc = kc.BatchedLayerCache.from_luts(4, Hkv, L + T, klut, vcent, device=dev, q_heads=Hq, batch=k)
    pc = kc.PagedLayerCache.from_luts(4, Hkv, klut, vcent, device=dev, q_heads=Hq, batch=k, page_size=P,
                                      n_pool=k * -(-(L + T) // P), max_pages=-(-(L + T) // P))
    g = torch.Generator(device=dev).manual_seed(1)
    rnd = lambda n: (torch.randn((n, Hkv * 128), generator=g, device=dev) * sigma + mu).half().float()   # noqa: E731
    for b in range(k):
        kk, vv = rnd(L), rnd(L)
        bc.seq(b).append_chunk(kk, vv)
        pc.append_chunk(b, kk, vv)
    bc.commit()
    pc.commit()
    slots, counts = list(range(k)), [T] * k
    K, V = rnd(k * T), rnd(k * T)
    q = torch.randn((k * T, Hq, 128), generator=g, device=dev) * 0.5
    rows = [slice(b * T, (b + 1) * T) for b in range(k)]
    parts = [(q[r].contiguous(), K[r].contiguous(), V[r].contiguous()) for r in rows]

    def reset():
        for b in range(k):
            bc.seq(b).len = L
            pc.pages.lens_host[b] = L

    def app_ragged():
        reset()
        bc.append_chunks(slots, K, V, counts)

    def app_loop():
        reset()
        for b, (_, kk, vv) in enumerate(parts):
            bc.seq(b).append_chunk(kk, vv)

    def papp_ragged():
        reset()
        pc.append_chunks(slots, K, V, counts)

    def papp_loop():
        reset()
        for b, (_, kk, vv) in enumerate(parts):
            pc.append_chunk(b, kk, vv)
    reset()
    att_ragged = lambda: bc.attend_chunks(slots, q, K, V, counts, rope_theta=THETA)   # noqa: E731

    def att_loop():
        for b, (qq, kk, vv) in enumerate(parts):
            bc.seq(b).attend_chunk_fused(qq, kk, vv, rope_theta=THETA)
    out = dict(shape="llama3_8b", heads=[Hq, Hkv], slots=k, T=T, L=L, page_size=P)
    for name, fr, fl in (("append_contiguous", app_ragged, app_loop), ("append_paged", papp_ragged, papp_loop),
                         ("attend_contiguous", att_ragged, att_loop)):
        ms_r, ms_l = events(fr, calls), events(fl, calls)
        out[name] = dict(ragged_ms=round(ms_r, 4), per_slot_sum_ms=round(ms_l, 4), ratio=round(ms_r / ms_l, 3))
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--layers", type=int, default=32)
    ap.add_argument("--reps", type=int, default=2)
    ap.add_argument("--calls", type=int, default=10)
    ap.add_argument("--page", type=int, default=640)
    ap.add_argument("--models", default="llama3_8b,llama7b")
    args = ap.parse_args()
    import torch
    dev = torch.device("cuda", 0)
    out = dict(gpu=gpu_info(0), page_size=args.page)

    def part(key, value):       # each part also goes to stderr as it completes
        out[key] = value
        print(json.dumps({key: value}), file=sys.stderr, flush=True)
        torch.cuda.empty_cache()
    part("kernels", measure_kernels(args.page, args.calls, dev))
    part("follow_up", measure_follow_up(args.layers, args.page, args.reps, dev))
    part("fork", measure_fork(args.layers, args.page, args.reps, dev))
    for m in args.models.split(","):
        part("grid_" + m, measure_grid(m, args.layers, args.page, args.reps, dev))
    print(json.dumps(out))


if __name__ == "__main__":
    main()
