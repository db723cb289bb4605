#!/usr/bin/env python
"""bench_resnet_glue.py -- where a denoising step of the default workload spends its time around the ResNet blocks.

    python bench_resnet_glue.py --out DIR [--steps 5]

Runs bench.py's default workload (aurora_1 map, SD1.5-shaped fp16 UNet, 512x512, LMS, CFG 7.5, CUDA graph, one image:
a batch-2 UNet forward per step), warms it up (graph capture, cuDNN autotune), then records --steps graph-replayed steps
under torch.profiler with CUDA activities, in a run of its own.  The Chrome trace goes to DIR/resnet_glue_trace.json.

Prints one JSON line: kernels per step, and per step the count and summed device time of each kernel family:
  broadcast_add   non-vectorised ATen add kernels (elementwise_kernel<128, 4, ...> with an add functor): the per-channel
                  conv-bias adds cuDNN leaves to `aten::_convolution` on channels-last outputs, among others
  vectorized_add  vectorised ATen adds (contiguous tensor + tensor, e.g. residual adds)
  resnet_residual the native ResNet-block epilogue (block input or shortcut + conv2 output + biases)
  group_norm      the native GroupNorm statistics and apply kernels
  convolution     cuDNN / CUTLASS convolution kernels (with their workspace-init kernels)
  other           everything else
cuDNN's autotuning picks its convolution kernels anew in every process, so the convolution row moves between runs of
the same code.
with the card's name, power limit and SM clocks.
"""
from __future__ import annotations

import argparse
import json
import os
import sys
from collections import defaultdict

import torch

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, ROOT)

import bench  # noqa: E402  (workload definition, device info)

FAMILIES = ("broadcast_add", "vectorized_add", "resnet_residual", "group_norm", "convolution", "other")


def family(name: str) -> str:
    n = name.lower()
    if "resnet_residual" in n:
        return "resnet_residual"
    if "gn_stats_kernel" in n or "gn_apply_kernel" in n:
        return "group_norm"
    if "add" in n and "elementwise_kernel" in n and "at::native" in n:
        return "vectorized_add" if "vectorized_elementwise_kernel" in n else "broadcast_add"
    if "sdpa" not in n and any(k in n for k in ("fprop", "conv", "implicit_gemm")):   # cuDNN's flash SDPA says fprop too
        return "convolution"
    return "other"


def summarize(trace_path: str, steps: int) -> dict:
    with open(trace_path) as f:
        events = json.load(f)["traceEvents"]
    kernels = [e for e in events if e.get("cat") == "kernel"]
    count, us = defaultdict(int), defaultdict(float)
    for e in kernels:
        fam = family(e["name"])
        count[fam] += 1
        us[fam] += float(e.get("dur", 0.0))
    return {"kernels_per_step": len(kernels) / steps,
            "kernel_us_per_step": sum(us.values()) / steps,
            "families": {f: {"launches_per_step": count[f] / steps, "us_per_step": us[f] / steps} for f in FAMILIES}}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", required=True, help="directory for the profiler trace")
    ap.add_argument("--steps", type=int, default=5)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_resnet_glue.py needs a CUDA device (H100)")
    import paint_with_words_sd_b200 as P
    from paint_with_words_sd_b200.pipeline import PwWSampler
    from paint_with_words_sd_b200.synthetic import RandomTextEncoder, SimpleWordTokenizer
    from torch.profiler import ProfilerActivity, profile

    os.makedirs(args.out, exist_ok=True)
    device = torch.device("cuda", 0)
    torch.cuda.set_device(device)
    torch.backends.cudnn.benchmark = True
    cfg = bench.CONFIGS[2]
    unet = bench.build_unet(bench.unet_config(cfg["unet"]), seed=0, dtype=torch.float16, device=device)
    unet = unet.to(memory_format=torch.channels_last)
    P.patch_unet(unet)
    sch = bench.LMSDiscreteScheduler(beta_start=0.00085, beta_end=0.012, beta_schedule="scaled_linear")
    sch.set_timesteps(cfg["sched_steps"])
    tok, enc = SimpleWordTokenizer(), RandomTextEncoder(cfg["text_dim"]).to(device)
    conds, unconds, lat0, extra = bench.build_images(cfg, device, [0], tok, enc, sch)
    smp = PwWSampler(unet, sch, conds, unconds, lat0, bench.weight_function, bench.GUIDANCE, extra_input=extra)
    trace = os.path.join(args.out, "resnet_glue_trace.json")
    try:
        with torch.no_grad():
            for _ in range(3):                           # graph capture, cuDNN autotune
                smp.step()
            torch.cuda.synchronize()
            with bench.ClockSampler(0) as clk, profile(activities=[ProfilerActivity.CPU, ProfilerActivity.CUDA]) as prof:
                for _ in range(args.steps):
                    smp.step()
                torch.cuda.synchronize()
            prof.export_chrome_trace(trace)
    finally:
        P.unpatch_all()
    line = {"metric": "resnet_glue_kernels_per_step", "unit": "kernels, us",
            "config": {"workload": cfg["what"], "profiled_steps": args.steps, "cuda_graph": True,
                       "native_launches_per_step": smp.native_launches_per_step},
            "device": bench.device_info(0), "clocks": clk.summary()}
    line.update(summarize(trace, args.steps))
    print(json.dumps(line), flush=True)


if __name__ == "__main__":
    main()
