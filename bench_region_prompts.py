#!/usr/bin/env python
"""bench_region_prompts.py -- the cost of region prompts: bench.py's default workload (aurora_1 map, SD1.5-shaped UNet,
512x512, LMS, CFG 7.5, fp16, one GPU) with 0, 1 and 2 region prompts, and the cross-attention kernel alone in region
mode against streaming mode.

    python bench_region_prompts.py [--steps 27] [--rounds 5] [--warmup 3] [--no-kernels]

One JSON line on stdout:
  steps_per_s  per region count R in {0, 1, 2}: the median over `rounds` of denoising steps/s (CUDA-graph replay,
               CUDA-event time); the three samplers are built once and timed in alternation, round by round.  R = 0 is
               the plain call (T = 77); R regions make a context of 1 + R chunks (T = 154, 231).
  kernel       per KC in {2, 3} at the N = 4096 level (8 heads of 40, cond + uncond, the cond image biased): one
               pww_xattn_fused_f16 launch (streaming softmax over all chunks) and one pww_xattn_fused_region_f16 launch
               (one softmax per chunk; the cond image's weights from two painted regions of the aurora_1 map, the uncond
               image on its first chunk alone), microseconds per launch, CUDA graph of back-to-back launches
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
from paint_with_words_sd_b200.conditioning import (_encode_text_color_inputs, pack_weight_map,  # noqa: E402
                                                   region_chunk_weights)
from paint_with_words_sd_b200.scheduler import LMSDiscreteScheduler  # noqa: E402
from paint_with_words_sd_b200.synthetic import RandomTextEncoder, SimpleWordTokenizer  # noqa: E402
from paint_with_words_sd_b200.unet import build_unet  # noqa: E402
from tests.fixtures import SETTINGS, color_map_image  # noqa: E402

SENTENCES = ["a bright green aurora over the snowy mountains", "a calm dark lake reflecting the stars"]


def regions(r: int) -> dict:
    colours = list(SETTINGS["aurora"]["ctx"])
    return {colours[i]: SENTENCES[i] for i in range(r)}


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
        for r in (0, 1, 2):
            sch = LMSDiscreteScheduler(beta_start=0.00085, beta_end=0.012, beta_schedule="scaled_linear")
            sch.set_timesteps(cfg["sched_steps"])
            seeds, sep, cond, uncond = _encode_text_color_inputs(
                enc, tok, device, color_map_image("aurora", size), dict(s["ctx"]), s["prompt"], "",
                region_prompts=regions(r) or None)
            lat0 = (initial_latents((1, 4, size // 8, size // 8), 0, seeds, sep) * sch.init_noise_sigma).to(device)
            runs[r] = (PwWSampler(unet, sch, [cond], [uncond], lat0, bench.weight_function, bench.GUIDANCE), lat0,
                       int(cond["CONTEXT_TENSOR"].shape[1]))

        def run(r, n):
            sampler, lat0, _ = runs[r]
            for _ in range(n):
                if sampler._step_no >= cfg["sched_steps"]:
                    sampler.restart(lat0)
                sampler.step()

        rates = {r: [] for r in runs}
        with torch.no_grad():
            for r in runs:
                run(r, warmup)
            for _ in range(rounds):
                for r in runs:
                    torch.cuda.synchronize(device)
                    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                    e0.record()
                    run(r, steps)
                    e1.record()
                    torch.cuda.synchronize(device)
                    rates[r].append(steps / (e0.elapsed_time(e1) / 1e3))
        return {f"R{r}": {"steps_per_s": float(np.median(v)), "all": v, "T": runs[r][2],
                          "native_launches_per_step": runs[r][0].native_launches_per_step} for r, v in rates.items()}
    finally:
        P.unpatch_all()


def kernel_us(device, kc: int, H=8, D=40, B=2, iters=64, reps=5, target_mb=192) -> dict:
    from paint_with_words_sd_b200 import _native
    L = _native.lib()
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
    rw = region_chunk_weights(color_map_image("aurora", 512), regions(kc - 1), 0.2, 8)[None].to(device).contiguous()
    idx = torch.tensor([0, -1], dtype=torch.int32, device=device)
    stats = torch.zeros(B, dtype=torch.float32, device=device)
    gs = torch.full((1,), 0.4 * math.log(8.0), dtype=torch.float32, device=device)
    fws = torch.zeros(L.pww_xattn_fused_workspace_bytes(), dtype=torch.uint8, device=device)

    def launch(region):
        def fn(i, stream):
            q, o = qs[i % nsets], outs[i % nsets]
            args = (q.data_ptr(), k.data_ptr(), v.data_ptr(), o.data_ptr(), B, H, N, T, D, q.stride(0), q.stride(1),
                    k.stride(0), k.stride(1), o.stride(0), o.stride(1), mp.data_ptr(), mp.stride(0), 1, ci.data_ptr(),
                    idx.data_ptr(), 0, gs.data_ptr(), D ** -0.5, stats.data_ptr(), fws.data_ptr(), fws.numel(), stream)
            if region:
                _native.check(L.pww_xattn_fused_region_f16(*args, rw.data_ptr(), rw.stride(0)), "region")
            else:
                _native.check(L.pww_xattn_fused_f16(*args), "fused")
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

    streaming, region = [], []
    for _ in range(3):                     # alternated
        streaming.append(timed(launch(False)))
        region.append(timed(launch(True)))
    return {"streaming_us": float(np.median(streaming)), "region_us": float(np.median(region)),
            "cond_rows_per_chunk": [int((rw[0, :, c] != 0).sum()) for c in range(kc)]}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=27)
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--no-kernels", action="store_true", help="loop only: skip the kernel timings")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_region_prompts.py needs a CUDA device (H100)")
    device = torch.device("cuda", 0)
    torch.cuda.set_device(device)
    torch.backends.cudnn.benchmark = True
    line = {"metric": bench.METRIC, "unit": bench.UNIT, "steps": args.steps, "rounds": args.rounds,
            "config": {"workload": bench.CONFIGS[2]["what"], "cuda_graph": True},
            "steps_per_s": loop_rates(device, args.steps, args.rounds, max(3, args.warmup))}
    if not args.no_kernels:
        line["kernel"] = {f"KC{kc}": kernel_us(device, kc) for kc in (2, 3)}
        line["kernel"]["note"] = "N=4096 C=320 H=8, B=2 (cond with region weights + uncond), cond biased"
    line["device"] = bench.device_info(0)
    print(json.dumps(line), flush=True)


if __name__ == "__main__":
    main()
