#!/usr/bin/env python
"""bench_groupnorm.py -- the native GroupNorm (`pww_groupnorm_nhwc_f16`) at every shape the default workload runs.

    python bench_groupnorm.py [--reps 32] [--iters 20] [--json FILE]

The default workload's step (bench.py: SD1.5-shaped fp16 UNet, 512x512, cond + uncond as one batch-2 forward) runs 61
GroupNorms, B = 2, G = 32, at the 14 (HW, C) shapes of SHAPES; `calls` is how many of them a step runs.  Each shape is
timed in three variants: SiLU with the per-channel `add` (a ResNet block's GroupNorm 2), SiLU alone (GroupNorm 1,
`conv_norm_out`) and plain (a transformer's), and in two input regimes:
  l2   one buffer set, as in the step, where the producer has just written the activation;
  hbm  buffer sets rotating over more than the 50 MB L2, so every pass reads and writes HBM.
CUDA events time a CUDA graph of --reps back-to-back calls, replayed --iters times.  A separate torch.profiler run of
the same graph splits the time into the statistics and apply kernels.  Bytes are the algorithm's: the activation read
twice and written once, 3*B*HW*C*2.  The weighted total is sum(calls * us) per variant.
"""
from __future__ import annotations

import argparse
import json
import os
import sys
import tempfile

import torch

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, ROOT)

import bench  # noqa: E402  (device info, clock sampler)

B, G = 2, 32
# (HW, C, calls per step)
SHAPES = [(4096, 320, 13), (4096, 640, 2), (4096, 960, 1),
          (1024, 320, 1), (1024, 640, 11), (1024, 960, 1), (1024, 1280, 1), (1024, 1920, 1),
          (256, 640, 1), (256, 1280, 11), (256, 1920, 1), (256, 2560, 2),
          (64, 1280, 12), (64, 2560, 3)]
VARIANTS = {"silu_add": (True, True), "silu": (True, False), "plain": (False, False)}
HBM_GBPS = 3350.0          # H100 SXM data sheet
L2_BYTES = 50 << 20


def _graph(L, HW, C, silu, with_add, nsets, reps, dev):
    g = torch.Generator(device="cpu").manual_seed(HW + C)
    xs = [(torch.randn(B, HW, C, generator=g) * 1.5 + 0.3).half().to(dev) for _ in range(nsets)]
    ys = [torch.empty_like(x) for x in xs]
    gamma = (torch.randn(C, generator=g) * 0.5 + 1.0).half().to(dev)
    beta = (torch.randn(C, generator=g) * 0.2).half().to(dev)
    add = (torch.randn(B, C, generator=g) * 0.5).half().to(dev) if with_add else None
    nbytes = L.pww_groupnorm_workspace_bytes(B, HW, G)
    ws = torch.zeros(max(nbytes, 256), dtype=torch.uint8, device=dev)

    def call(i):
        rc = L.pww_groupnorm_nhwc_f16(xs[i % nsets].data_ptr(), None if add is None else add.data_ptr(), C,
                                      gamma.data_ptr(), beta.data_ptr(), ys[i % nsets].data_ptr(), B, HW, C, G, 1e-5,
                                      1 if silu else 0, ws.data_ptr(), ws.numel(), torch.cuda.current_stream().cuda_stream)
        assert rc == 0, rc

    for i in range(nsets):
        call(i)
    torch.cuda.synchronize()
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        for i in range(reps):
            call(i)
    graph.replay()
    torch.cuda.synchronize()
    return graph, (xs, ys, gamma, beta, add, ws)


def _time(graph, iters, reps):
    for _ in range(3):
        graph.replay()
    t0, t1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    t0.record()
    for _ in range(iters):
        graph.replay()
    t1.record()
    t1.synchronize()
    return t0.elapsed_time(t1) * 1e3 / (iters * reps)


def _split(graph, reps, tmp):
    """us per call of the statistics and the apply kernel, from a profiled replay."""
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(4):
            graph.replay()
        torch.cuda.synchronize()
    path = os.path.join(tmp, "gn_trace.json")
    prof.export_chrome_trace(path)
    with open(path) as f:
        kernels = [e for e in json.load(f)["traceEvents"] if e.get("cat") == "kernel"]
    st = sum(float(e["dur"]) for e in kernels if "gn_stats_kernel" in e["name"])
    ap = sum(float(e["dur"]) for e in kernels if "gn_apply_kernel" in e["name"])
    return st / (4 * reps), ap / (4 * reps)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=32, help="calls per captured graph")
    ap.add_argument("--iters", type=int, default=20, help="timed replays of the graph")
    ap.add_argument("--json", default=None, help="also write the results to this file")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_groupnorm.py needs a CUDA device (H100)")
    from paint_with_words_sd_b200 import _native
    L = _native.lib()
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    rows, totals = [], {}
    print(f"{'regime':6} {'variant':8} {'HW':>5} {'C':>5} {'calls':>5} {'us':>8} {'stats':>7} {'apply':>7} "
          f"{'MB':>6} {'GB/s':>7} {'of HBM':>6}")
    with tempfile.TemporaryDirectory() as tmp, bench.ClockSampler(0) as clk:
        for regime in ("l2", "hbm"):
            for variant, (silu, with_add) in VARIANTS.items():
                tot = 0.0
                for HW, C, calls in SHAPES:
                    act = B * HW * C * 2
                    nsets = 1 if regime == "l2" else max(2, -(-4 * L2_BYTES // (2 * act)))
                    reps = max(args.reps, nsets)          # one graph visits every set
                    graph, keep = _graph(L, HW, C, silu, with_add, nsets, reps, dev)
                    us = _time(graph, args.iters, reps)
                    st, apl = _split(graph, reps, tmp)
                    del graph, keep
                    nbytes = 3 * act
                    gbps = nbytes / us * 1e-3
                    tot += calls * us
                    rows.append({"regime": regime, "variant": variant, "HW": HW, "C": C, "calls": calls, "us": us,
                                 "stats_us": st, "apply_us": apl, "bytes": nbytes, "GBps": gbps,
                                 "hbm_fraction": gbps / HBM_GBPS})
                    print(f"{regime:6} {variant:8} {HW:5d} {C:5d} {calls:5d} {us:8.2f} {st:7.2f} {apl:7.2f} "
                          f"{nbytes / 1e6:6.2f} {gbps:7.0f} {gbps / HBM_GBPS:6.1%}", flush=True)
                totals[f"{regime}/{variant}"] = tot
                print(f"{regime:6} {variant:8} weighted total per step (sum calls * us): {tot:.1f} us", flush=True)
    line = {"metric": "groupnorm_us", "B": B, "G": G, "device": bench.device_info(0), "clocks": clk.summary(),
            "weighted_us_per_step": totals, "shapes": rows}
    if args.json:
        with open(args.json, "w") as f:
            json.dump(line, f, indent=1)
    print(json.dumps({k: line[k] for k in ("metric", "device", "clocks", "weighted_us_per_step")}), flush=True)


if __name__ == "__main__":
    main()
