#!/usr/bin/env python
"""bench_negative_regions.py -- the cost of negative region prompts: bench.py's default workload (aurora_1 map,
SD1.5-shaped UNet, 512x512, LMS, CFG 7.5, fp16, one GPU) with two region prompts, without and with a negative sentence
for both regions, and the cross-attention kernel alone with the uncond rows on their first chunk against weighted.

    python bench_negative_regions.py [--steps 27] [--rounds 5] [--warmup 3] [--no-kernels]

One JSON line on stdout:
  steps_per_s  "regions" (region_prompts alone: the uncond images on chunk 0) and "negatives" (the same call with
               negative_region_prompts for both colours: the uncond images weigh their own sentences): the median over
               `rounds` of denoising steps/s (CUDA-graph replay, CUDA-event time); both samplers are built once and
               timed in alternation, round by round.  Both contexts are T = 231.
  kernel       per batch of B in {2, 16} images (B / 2 cond images, biased, with the aurora_1 map's region weights, and
               B / 2 uncond images) at the N = 4096 level (8 heads of 40, T = 231): one pww_xattn_fused_region_rows_f16
               launch with the uncond rows on chunk 0 (region_index -1) and one with them weighted by the negative
               side's weights, microseconds per launch, CUDA graph of back-to-back launches, alternated
  device       name and power limit of the GPU the numbers were measured on
Writes nothing.
"""
from __future__ import annotations

import argparse
import json
import math
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, ROOT)

import bench  # noqa: E402  (workload definition, device info)
from bench_region_prompts import SENTENCES, regions  # noqa: E402
from paint_with_words_sd_b200.conditioning import (_encode_text_color_inputs, pack_weight_map,  # noqa: E402
                                                   region_chunk_weights)
from paint_with_words_sd_b200.scheduler import LMSDiscreteScheduler  # noqa: E402
from paint_with_words_sd_b200.synthetic import RandomTextEncoder, SimpleWordTokenizer  # noqa: E402
from paint_with_words_sd_b200.unet import build_unet  # noqa: E402
from tests.fixtures import SETTINGS, color_map_image  # noqa: E402

NEGATIVES = ["a blurry washed-out sky", "rough water with waves"]


def negatives() -> dict:
    colours = list(SETTINGS["aurora"]["ctx"])
    return {colours[i]: NEGATIVES[i] for i in range(len(SENTENCES))}


def loop_rates(device, steps: int, rounds: int, warmup: int) -> dict:
    import paint_with_words_sd_b200 as P
    from paint_with_words_sd_b200.pipeline import PwWSampler, initial_latents
    cfg = bench.CONFIGS[2]
    size = cfg["size"]
    unet = build_unet(bench.unet_config(cfg["unet"]), seed=0, dtype=torch.float16, device=device)
    unet = unet.to(memory_format=torch.channels_last)
    P.patch_unet(unet)
    try:
        tok, enc = SimpleWordTokenizer(), RandomTextEncoder(cfg["text_dim"]).to(device)
        s = SETTINGS["aurora"]
        runs = {}
        for name, neg in (("regions", None), ("negatives", negatives())):
            sch = LMSDiscreteScheduler(beta_start=0.00085, beta_end=0.012, beta_schedule="scaled_linear")
            sch.set_timesteps(cfg["sched_steps"])
            seeds, sep, cond, uncond = _encode_text_color_inputs(
                enc, tok, device, color_map_image("aurora", size), dict(s["ctx"]), s["prompt"], "",
                region_prompts=regions(2), negative_region_prompts=neg)
            lat0 = (initial_latents((1, 4, size // 8, size // 8), 0, seeds, sep) * sch.init_noise_sigma).to(device)
            runs[name] = (PwWSampler(unet, sch, [cond], [uncond], lat0, bench.weight_function, bench.GUIDANCE), lat0,
                          int(cond["CONTEXT_TENSOR"].shape[1]))

        def run(name, n):
            sampler, lat0, _ = runs[name]
            for _ in range(n):
                if sampler._step_no >= cfg["sched_steps"]:
                    sampler.restart(lat0)
                sampler.step()

        rates = {name: [] for name in runs}
        with torch.no_grad():
            for name in runs:
                run(name, warmup)
            for _ in range(rounds):
                for name in runs:
                    torch.cuda.synchronize(device)
                    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                    e0.record()
                    run(name, steps)
                    e1.record()
                    torch.cuda.synchronize(device)
                    rates[name].append(steps / (e0.elapsed_time(e1) / 1e3))
        return {name: {"steps_per_s": float(np.median(v)), "all": v, "T": runs[name][2],
                       "native_launches_per_step": runs[name][0].native_launches_per_step}
                for name, v in rates.items()}
    finally:
        P.unpatch_all()


def kernel_us(device, B: int, H=8, D=40, iters=64, reps=5, target_mb=192) -> dict:
    from paint_with_words_sd_b200 import _native
    L = _native.lib()
    m, kc = B // 2, 3
    N, C, T = 4096, H * D, 77 * kc
    g = torch.Generator().manual_seed(0)
    nsets = max(2, int(math.ceil(target_mb * 1e6 / (B * N * C * 4))))     # buffer sets larger than L2
    qs = [(torch.randn(B, N, C, generator=g) * 0.5).half().to(device) for _ in range(nsets)]
    outs = [torch.empty(B, N, C, dtype=torch.float16, device=device) for _ in range(nsets)]
    k = (torch.randn(B, T, C, generator=g) * 0.5).half().to(device)
    v = (torch.randn(B, T, C, generator=g) * 0.5).half().to(device)
    w = torch.zeros(1, N, T)
    w[0, :, 3:5] = torch.rand(N, 1, generator=g) > 0.5
    mp, ci = (t.to(device) for t in pack_weight_map(w))
    cmap = color_map_image("aurora", 512)
    rw = torch.stack([region_chunk_weights(cmap, regions(2), 0.2, 8),
                      region_chunk_weights(cmap, negatives(), 0.2, 8)], 0).to(device).contiguous()
    widx = torch.tensor([0] * m + [-1] * m, dtype=torch.int32, device=device)
    rows = {"uncond_chunk0": torch.tensor([0] * m + [-1] * m, dtype=torch.int32, device=device),
            "uncond_weighted": torch.tensor([0] * m + [1] * m, dtype=torch.int32, device=device)}
    stats = torch.zeros(B, dtype=torch.float32, device=device)
    gs = torch.full((1,), 0.4 * math.log(8.0), dtype=torch.float32, device=device)
    fws = torch.zeros(L.pww_xattn_fused_workspace_bytes(), dtype=torch.uint8, device=device)

    def launch(ridx):
        def fn(i, stream):
            q, o = qs[i % nsets], outs[i % nsets]
            rc = L.pww_xattn_fused_region_rows_f16(
                q.data_ptr(), k.data_ptr(), v.data_ptr(), o.data_ptr(), B, H, N, T, D, q.stride(0), q.stride(1),
                k.stride(0), k.stride(1), o.stride(0), o.stride(1), mp.data_ptr(), mp.stride(0), 1, ci.data_ptr(),
                widx.data_ptr(), 0, gs.data_ptr(), D ** -0.5, stats.data_ptr(), fws.data_ptr(), fws.numel(), stream,
                rw.data_ptr(), rw.stride(0), ridx.data_ptr(), None)
            _native.check(rc, "region_rows")
        return fn

    def timed(fn):
        s = torch.cuda.Stream(device=device)
        with torch.cuda.stream(s):
            for i in range(3):
                fn(i, s.cuda_stream)
        s.synchronize()
        graph = torch.cuda.CUDAGraph()
        with torch.cuda.graph(graph, stream=s):
            for i in range(iters):
                fn(i, torch.cuda.current_stream(device).cuda_stream)
        t = []
        for _ in range(reps):
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            torch.cuda.synchronize(device)
            e0.record()
            graph.replay()
            e1.record()
            torch.cuda.synchronize(device)
            t.append(e0.elapsed_time(e1) * 1e3 / iters)
        return float(np.median(t))

    times = {name: [] for name in rows}
    for _ in range(3):                     # alternated
        for name, ridx in rows.items():
            times[name].append(timed(launch(ridx)))
    out = {f"{name}_us": float(np.median(t)) for name, t in times.items()}
    out["uncond_rows_per_chunk"] = [int((rw[1, :, c] != 0).sum()) for c in range(kc)]
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=27)
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--no-kernels", action="store_true", help="loop only: skip the kernel timings")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_negative_regions.py needs a CUDA device (H100)")
    device = torch.device("cuda", 0)
    torch.cuda.set_device(device)
    torch.backends.cudnn.benchmark = True
    line = {"metric": bench.METRIC, "unit": bench.UNIT, "steps": args.steps, "rounds": args.rounds,
            "config": {"workload": bench.CONFIGS[2]["what"], "cuda_graph": True},
            "steps_per_s": loop_rates(device, args.steps, args.rounds, max(3, args.warmup))}
    if not args.no_kernels:
        line["kernel"] = {f"B{b}": kernel_us(device, b) for b in (2, 16)}
        line["kernel"]["note"] = "N=4096 C=320 H=8 T=231, B/2 cond (biased, region weights) + B/2 uncond"
    line["device"] = bench.device_info(0)
    print(json.dumps(line), flush=True)


if __name__ == "__main__":
    main()
