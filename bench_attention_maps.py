#!/usr/bin/env python
"""bench_attention_maps.py -- what attention recording costs.

    python bench_attention_maps.py [--steps 27] [--warmup 3] [--rounds 3] [--json FILE]

1. The default workload of bench.py (SD1.5-shaped fp16 UNet, 512x512, aurora colour map, cond + uncond as one batch-2
   forward, CUDA graph per step) in steps/s, with and without `PwWSampler(record_attention=True)`, the two samplers
   alternated in one process for --rounds rounds of --steps timed steps each (host clock around device-synchronised
   steps).
2. The cross-attention kernel alone at the top SD1.5 level (N = 4096, 8 heads of 40, T = 77), plain (`_multi`) against
   recording (`_rec`, every cond image recorded), for the cond + uncond batch (B = 2) and for 8 cond + 8 uncond images
   (B = 16): CUDA events around a CUDA graph of --reps back-to-back calls.
Prints one JSON object with the device name and power limit.
"""
from __future__ import annotations

import argparse
import json
import math
import os
import sys
import time

import torch

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, ROOT)

import bench  # noqa: E402  (workload set-up, device info)
import paint_with_words_sd_b200 as P  # noqa: E402
from paint_with_words_sd_b200 import attention  # noqa: E402
from paint_with_words_sd_b200.pipeline import PwWSampler  # noqa: E402
from paint_with_words_sd_b200.scheduler import LMSDiscreteScheduler  # noqa: E402
from paint_with_words_sd_b200.synthetic import RandomTextEncoder, SimpleWordTokenizer  # noqa: E402
from paint_with_words_sd_b200.unet import build_unet  # noqa: E402


def steps_per_s(args, dev) -> dict:
    cfg = bench.CONFIGS[2]                      # the default workload
    unet = build_unet(bench.unet_config(cfg["unet"]), seed=0, dtype=torch.float16, device=dev)
    P.patch_unet(unet)
    tok, enc = SimpleWordTokenizer(), RandomTextEncoder(cfg["text_dim"]).to(dev)
    sch = LMSDiscreteScheduler(beta_start=0.00085, beta_end=0.012, beta_schedule="scaled_linear")
    sch.set_timesteps(cfg["sched_steps"])
    wf = bench.make_weight_function(cfg["coef"])
    samplers = {}
    for rec in (False, True):
        conds, unconds, lat, _ = bench.build_images(cfg, dev, [0], tok, enc, sch)
        samplers[rec] = (PwWSampler(unet, sch, conds, unconds, lat, wf, bench.GUIDANCE, record_attention=rec), lat)
    n = args.warmup + args.steps
    if n > len(sch.timesteps):
        raise SystemExit(f"--warmup + --steps must be at most {len(sch.timesteps)}")
    rates = {False: [], True: []}
    for _ in range(args.rounds):
        for rec, (s, lat) in samplers.items():
            s.restart(lat)
            s.run(args.warmup)
            torch.cuda.synchronize(dev)
            t0 = time.perf_counter()
            s.run(args.steps)
            torch.cuda.synchronize(dev)
            rates[rec].append(args.steps / (time.perf_counter() - t0))
    maps = samplers[True][0].attention_maps()[0]
    P.unpatch_all()
    med = {k: sorted(v)[len(v) // 2] for k, v in rates.items()}
    return {"plain_steps_per_s": rates[False], "record_steps_per_s": rates[True],
            "plain_median": med[False], "record_median": med[True],
            "record_cost_pct": 100.0 * (med[False] / med[True] - 1.0),
            "launches_per_step": {"plain": samplers[False][0].native_launches_per_step,
                                  "record": samplers[True][0].native_launches_per_step},
            "maps_finite": bool(torch.isfinite(maps).all())}


def kernel_us(dev, B, reps, iters, N=4096, H=8, D=40, T=77) -> dict:
    g = torch.Generator().manual_seed(B)
    q = (torch.randn(B, N, H * D, generator=g) * 0.5).half().to(dev)
    k = (torch.randn(B, T, H * D, generator=g) * 0.5).half().to(dev)
    v = (torch.randn(B, T, H * D, generator=g) * 0.5).half().to(dev)
    m = B // 2
    w = bench.region_weight_map(N).expand(m, N, T).contiguous().to(dev)
    idx = torch.tensor(list(range(m)) + [-1] * m, dtype=torch.int32, device=dev)
    kinds = torch.zeros(B, dtype=torch.int32, device=dev)
    gs = torch.full((B,), 0.4 * math.log(8.0), dtype=torch.float32, device=dev)
    ridx = torch.randint(-1, 5, (m, 80), generator=g).to(torch.int8).to(dev)
    acc = torch.zeros(m, H, N, 16, dtype=torch.float32, device=dev)
    stats = torch.zeros(64, dtype=torch.float32, device=dev)
    ws = torch.zeros(P._native.lib().pww_xattn_fused_workspace_bytes(), dtype=torch.uint8, device=dev)
    packed = attention._state(dev).packed(w)
    out = {}
    for name, record in (("plain", None), ("record", (ridx, idx, acc))):
        def call():
            attention.cross_attention(q, k, v, H, D ** -0.5, w, idx, kinds, gs, packed=packed, stats_out=stats,
                                      workspace=ws, record=record)
        for _ in range(3):
            call()
        torch.cuda.synchronize(dev)
        graph = torch.cuda.CUDAGraph()
        with torch.cuda.graph(graph):
            for _ in range(reps):
                call()
        graph.replay()
        torch.cuda.synchronize(dev)
        times = []
        for _ in range(iters):
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            graph.replay()
            e1.record()
            e1.synchronize()
            times.append(e0.elapsed_time(e1) * 1e3 / reps)
        out[name] = sorted(times)[len(times) // 2]
    out["record_cost_pct"] = 100.0 * (out["record"] / out["plain"] - 1.0)
    out["acc_bytes_per_call"] = 2 * m * H * N * 16 * 4          # read + write of the accumulator
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=27)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--reps", type=int, default=64)
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--json", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_attention_maps.py measures on a GPU; none is available")
    dev = torch.device("cuda", 0)
    res = {"device": bench.device_info(0), "e2e": steps_per_s(args, dev),
           "kernel_us": {f"B{B}": kernel_us(dev, B, args.reps, args.iters) for B in (2, 16)}}
    line = json.dumps(res)
    print(line)
    if args.json:
        with open(args.json, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
