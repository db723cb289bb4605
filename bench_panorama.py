#!/usr/bin/env python
"""bench_panorama.py -- what a MultiDiffusion panorama costs: whole 512x2048 panoramas at two strides and two view
batch sizes, and the canvas update launch alone against the same tail written as torch ops.

    python bench_panorama.py [--reps 3] [--steps 30] [--no-loop] [--no-update]

Loop: the SD1.5-shaped UNet (synthetic:sd15, seeded random weights), fp16, LMS, CFG 7.5, 30 steps, on a 512x2048
colour map (four fixture maps side by side: a 64x256 latent canvas) with 64x64 windows: stride 8 (25 windows) and
stride 16 (13 windows), view_batch_size 16 and 32.  Each PanoramaSampler is timed whole with CUDA events after a
warm-up run (graph capture, library autotune), the configurations alternated over --reps rounds: the median and range
of steps/s and seconds per panorama, and the native launches per step.

Update: at 25 windows (stride 8) with fp16 channels-last window outputs in one chunk, an LMS step with a full history
ring: pww_window_update against the torch ops of the same tail (per window: crop, CFG, ordered scatter-add; then the
divide and the step form), each captured in a CUDA graph of --iters steps, alternated, microseconds per step; and
whether the two give the same bits from the same state.

One JSON line on stdout, with the GPU's name and power limit.  Writes nothing.
"""
from __future__ import annotations

import argparse
import ctypes
import functools
import json
import os
import sys

import numpy as np
import torch
from PIL import Image

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, ROOT)

import bench  # noqa: E402  (device info, weight function)
from paint_with_words_sd_b200 import _native  # noqa: E402
from paint_with_words_sd_b200 import panorama as PN  # noqa: E402
from paint_with_words_sd_b200.pipeline import _BETA  # noqa: E402
from paint_with_words_sd_b200.scheduler import LMSDiscreteScheduler  # noqa: E402
from paint_with_words_sd_b200.synthetic import RandomTextEncoder, SimpleWordTokenizer  # noqa: E402
from paint_with_words_sd_b200.unet import UNetConfig, build_unet  # noqa: E402
from tests.fixtures import SETTINGS, color_map_image  # noqa: E402

KW = dict(beta_start=0.00085, beta_end=0.012, beta_schedule="scaled_linear")
HEIGHT, WIDTH, WINDOW = 512, 2048, 64
STRIDES, VIEW_BATCHES = (8, 16), (16, 32)


def _events_ms(fn) -> float:
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    e0.record()
    fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1)


def color_map() -> Image.Image:
    out = Image.new("RGB", (WIDTH, HEIGHT))
    for i, name in enumerate(("aurora", "cat_dog", "aurora", "cat_dog")):
        out.paste(color_map_image(name, HEIGHT), (i * HEIGHT, 0))
    return out


def _full_run(smp, lat, steps):
    smp.restart(lat)
    for _ in range(steps):
        smp.step()


def loop(device, steps: int, reps: int) -> dict:
    import paint_with_words_sd_b200 as P
    cfg = UNetConfig.sd15()
    unet = build_unet(cfg, seed=0, dtype=torch.float16, device=device).to(memory_format=torch.channels_last)
    P.patch_unet(unet)
    try:
        tok, enc = SimpleWordTokenizer(), RandomTextEncoder(cfg.cross_attention_dim).to(device)
        s = SETTINGS["aurora"]
        cm = color_map()
        lat = (PN.panorama_latents(cm, dict(s["ctx"]), tok, 0) * 14.6).to(device)
        runs = {}
        for stride in STRIDES:
            views = PN.panorama_views(HEIGHT // 8, WIDTH // 8, WINDOW, stride)
            conds, unconds = PN.panorama_conditioning(enc, tok, device, cm, dict(s["ctx"]), s["prompt"], "", views,
                                                      WINDOW)
            for vbs in VIEW_BATCHES:
                sch = LMSDiscreteScheduler(**KW)
                sch.set_timesteps(steps)
                smp = PN.PanoramaSampler(unet, sch, conds, unconds, lat, views, WINDOW, bench.weight_function, 7.5,
                                         view_batch_size=vbs)
                run = functools.partial(_full_run, smp, lat, steps)
                run()                                           # warm-up: graph capture, library autotune
                runs[f"stride{stride}_vbs{vbs}"] = (smp, run, len(views[0]) * len(views[1]))
            del conds, unconds
        times = {k: [] for k in runs}
        for _ in range(reps):                                   # alternated: drift of the card hits every config
            for k, (_, run, _) in runs.items():
                times[k].append(_events_ms(run))
        res = {}
        for k, (smp, _, views) in runs.items():
            t = times[k]
            res[k] = {"windows": views, "chunks": len(smp._firsts), "steps_per_s": steps / (float(np.median(t)) / 1e3),
                      "steps_per_s_range": [steps / (max(t) / 1e3), steps / (min(t) / 1e3)],
                      "s_per_panorama": float(np.median(t)) / 1e3,
                      "native_launches_per_step": smp.native_launches_per_step,
                      "finite": bool(torch.isfinite(smp.latents).all())}
        return res
    finally:
        P.unpatch_all()


def update(device, iters: int, reps: int) -> dict:
    L = _native.lib()
    H, W, win = HEIGHT // 8, WIDTH // 8, WINDOW
    rows, cols = PN.panorama_views(H, W, win, 8)
    V = len(rows) * len(cols)
    g = torch.Generator().manual_seed(0)
    lat0 = (torch.randn(1, 4, H, W, generator=g) * 14.6).to(device)
    eps = torch.randn(2 * V, 4, win, win, generator=g).half().to(device).contiguous(memory_format=torch.channels_last)
    gscale = torch.tensor([7.5], device=device)
    step_row = torch.zeros(_BETA + 4, device=device)
    step_row[_BETA:] = torch.tensor([0.5, -0.2, 0.1, -0.05])
    form = torch.tensor([1.0, 0.0, 1.0, 0.0, 0.0, 0.0], device=device)      # LMS: q = eps, slot 0
    starts = (torch.tensor(rows, dtype=torch.int32, device=device), torch.tensor(cols, dtype=torch.int32, device=device))
    state = {k: (lat0.clone(), torch.zeros(4, 1, 4, H, W, device=device)) for k in ("native", "torch")}
    table = (ctypes.c_void_p * 1)(eps.data_ptr())

    def native():
        lat, hist = state["native"]
        _native.check(L.pww_window_update(table, 1, V, _native.PWW_DTYPE_F16, *eps.stride(), starts[0].data_ptr(),
                                          len(rows), starts[1].data_ptr(), len(cols), win, lat.data_ptr(),
                                          hist.data_ptr(), 4, None, gscale.data_ptr(), step_row[_BETA:].data_ptr(),
                                          form.data_ptr(), H, W, torch.cuda.current_stream(device).cuda_stream),
                      "pww_window_update")

    col_idx = [torch.arange(c, c + win, device=device) % W for c in cols]
    wins = [(r0, ci) for r0 in rows for ci in col_idx]
    beta = [0.5, -0.2, 0.1, -0.05]

    def torch_tail():                                           # the same arithmetic in the same order
        lat, hist = state["torch"]
        total, count = torch.zeros_like(lat), torch.zeros_like(lat)
        e = eps.float()
        for v, (r0, ci) in enumerate(wins):
            gv = e[V + v] + gscale * (e[v] - e[V + v])
            seen = count[0, :, r0:r0 + win, ci] > 0
            total[0, :, r0:r0 + win, ci] = torch.where(seen, total[0, :, r0:r0 + win, ci] + gv, gv)
            count[0, :, r0:r0 + win, ci] += 1
        q = 1.0 * (total / count)
        hist[0].copy_(q)
        acc = beta[0] * q
        for j in range(1, 4):
            acc = acc + beta[j] * hist[4 - j]
        lat.copy_(lat + acc)

    # one step of each from the same state: the same bits
    native()
    torch_tail()
    torch.cuda.synchronize()
    same = bool(torch.equal(state["native"][0], state["torch"][0]) and torch.equal(state["native"][1],
                                                                                  state["torch"][1]))
    diff = float((state["native"][0] - state["torch"][0]).abs().max())

    def graph_of(fn):
        s = torch.cuda.Stream(device=device)
        s.wait_stream(torch.cuda.current_stream(device))
        with torch.cuda.stream(s):
            for _ in range(2):
                fn()
        s.synchronize()
        graph = torch.cuda.CUDAGraph()
        with torch.cuda.graph(graph, stream=s):
            for _ in range(iters):
                fn()
        return graph

    graphs = {"native": graph_of(native), "torch": graph_of(torch_tail)}
    times = {k: [] for k in graphs}
    for _ in range(reps):                                       # alternated
        for k, gr in graphs.items():
            state[k][0].copy_(lat0)                             # keep the latents finite over the rounds
            state[k][1].zero_()
            times[k].append(_events_ms(gr.replay) * 1e3 / iters)
    return {"windows": V, "window_update_us": float(np.median(times["native"])),
            "torch_ops_us": float(np.median(times["torch"])), "same_bits": same, "max_abs_diff": diff}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=30)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--iters", type=int, default=50)
    ap.add_argument("--no-loop", action="store_true")
    ap.add_argument("--no-update", action="store_true")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_panorama.py needs a CUDA device (H100)")
    device = torch.device("cuda", 0)
    torch.cuda.set_device(device)
    torch.backends.cudnn.benchmark = True
    line = {"metric": "panorama_steps_per_sec_512x2048", "unit": "steps/s, s per panorama, us per launch",
            "config": {"workload": f"synthetic:sd15 {HEIGHT}x{WIDTH}, window {WINDOW}, strides {list(STRIDES)}, "
                                   f"view_batch_size {list(VIEW_BATCHES)}, LMS, {args.steps} steps, fp16, CFG 7.5, "
                                   "CUDA graph", "reps": args.reps},
            "device": bench.device_info(0)}
    with torch.no_grad():
        if not args.no_loop:
            line["loop"] = loop(device, args.steps, args.reps)
        if not args.no_update:
            line["update"] = update(device, args.iters, 5)
    print(json.dumps(line), flush=True)


if __name__ == "__main__":
    main()
