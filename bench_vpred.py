#!/usr/bin/env python
"""bench_vpred.py -- what guidance rescale costs: a v-prediction SD2.1 run at 768x768 with and without it, and the
sampler update launch alone, plain against rescale.

    python bench_vpred.py [--reps 5] [--steps 30] [--no-loop] [--no-update]

Loop: the SD2.1-shaped UNet (synthetic:sd21, seeded random weights) at 768x768 (96x96 latents), the aurora colour map,
one image, LMS with prediction_type="v_prediction" at 30 steps, fp16, CFG 7.5, CUDA-graph replay.  Two samplers, one with
guidance_rescale 0 (pww_sampler_update) and one with 0.7 (pww_sampler_update_rescale), are timed whole with CUDA events
after a warm-up run (graph capture), alternated over --reps rounds; each gets the median and the range of steps/s.

Update: the update launch alone at 64x64 and 96x96 latents, m = 1 and 8, fp16 channels-last UNet output, an LMS step
form with a full history ring: microseconds per launch from CUDA events over a CUDA graph of 200 back-to-back launches,
plain against rescale.

One JSON line on stdout, with the GPU's name and power limit.  Writes nothing.
"""
from __future__ import annotations

import argparse
import functools
import json
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, ROOT)

import bench  # noqa: E402  (device info, weight function)
from paint_with_words_sd_b200 import _native  # noqa: E402
from paint_with_words_sd_b200.conditioning import _encode_text_color_inputs  # noqa: E402
from paint_with_words_sd_b200.scheduler import LMSDiscreteScheduler  # noqa: E402
from paint_with_words_sd_b200.synthetic import RandomTextEncoder, SimpleWordTokenizer  # noqa: E402
from paint_with_words_sd_b200.unet import UNetConfig, build_unet  # noqa: E402
from tests.fixtures import SETTINGS, color_map_image  # noqa: E402

KW = dict(beta_start=0.00085, beta_end=0.012, beta_schedule="scaled_linear", prediction_type="v_prediction")
SIZE = 768
PHIS = (0.0, 0.7)


def _events_ms(fn) -> float:
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    e0.record()
    fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1)


def _full_run(smp, lat, steps):
    smp.restart(lat)
    for _ in range(steps):
        smp.step()


def loop(device, steps: int, reps: int) -> dict:
    import paint_with_words_sd_b200 as P
    from paint_with_words_sd_b200.pipeline import PwWSampler, initial_latents
    cfg = UNetConfig.sd21()
    unet = build_unet(cfg, seed=0, dtype=torch.float16, device=device).to(memory_format=torch.channels_last)
    P.patch_unet(unet)
    try:
        tok, enc = SimpleWordTokenizer(), RandomTextEncoder(cfg.cross_attention_dim).to(device)
        s = SETTINGS["aurora"]
        seeds, sep, cond, uncond = _encode_text_color_inputs(enc, tok, device, color_map_image("aurora", SIZE),
                                                             dict(s["ctx"]), s["prompt"], "")
        runs = {}
        for phi in PHIS:
            sch = LMSDiscreteScheduler(**KW)
            sch.set_timesteps(steps)
            lat = (initial_latents((1, 4, SIZE // 8, SIZE // 8), 0, seeds, sep) * sch.init_noise_sigma).to(device)
            smp = PwWSampler(unet, sch, [cond], [uncond], lat, bench.weight_function, 7.5, guidance_rescale=phi)
            run = functools.partial(_full_run, smp, lat, steps)
            run()                                               # warm-up: graph capture, library autotune
            runs[phi] = (smp, run)
        times = {phi: [] for phi in PHIS}
        for _ in range(reps):                                   # alternated: drift of the card hits both
            for phi in PHIS:
                times[phi].append(_events_ms(runs[phi][1]))
        res = {}
        for phi in PHIS:
            t = times[phi]
            res[f"phi{phi}"] = {"steps_per_s": steps / (float(np.median(t)) / 1e3),
                                "steps_per_s_range": [steps / (max(t) / 1e3), steps / (min(t) / 1e3)],
                                "ms_per_run": float(np.median(t)),
                                "native_launches_per_step": runs[phi][0].native_launches_per_step,
                                "finite": bool(torch.isfinite(runs[phi][0].latents).all())}
        return res
    finally:
        P.unpatch_all()


def update(device, m: int, hw: int, iters: int = 200, reps: int = 5) -> dict:
    L = _native.lib()
    g = torch.Generator().manual_seed(0)
    lat = (torch.randn(m, 4, hw, hw, generator=g) * 14.6).to(device)
    eps = torch.randn(2 * m, 4, hw, hw, generator=g).half().to(device).contiguous(memory_format=torch.channels_last)
    gscale = torch.full((m,), 7.5, device=device)
    phi = torch.full((m,), 0.7, device=device)
    beta = torch.tensor([0.5, -0.2, 0.1, -0.05], device=device)
    sigma = 14.6          # the v form of the LMS identity form at this sigma
    form = torch.tensor([1.0, sigma / (sigma ** 2 + 1), 1 / (sigma ** 2 + 1) ** 0.5, 0.0, 0.0, 0.0], device=device)
    hist = torch.zeros(4, m, 4, hw, hw, device=device)

    def plain():
        stream = torch.cuda.current_stream(device).cuda_stream
        _native.check(L.pww_sampler_update(eps.data_ptr(), _native.PWW_DTYPE_F16, *eps.stride(), lat.data_ptr(),
                                           hist.data_ptr(), 4, None, gscale.data_ptr(), beta.data_ptr(),
                                           form.data_ptr(), m, hw, hw, stream), "pww_sampler_update")

    def rescale():
        stream = torch.cuda.current_stream(device).cuda_stream
        _native.check(L.pww_sampler_update_rescale(eps.data_ptr(), _native.PWW_DTYPE_F16, *eps.stride(),
                                                   lat.data_ptr(), hist.data_ptr(), 4, None, gscale.data_ptr(),
                                                   beta.data_ptr(), form.data_ptr(), phi.data_ptr(), None, m, hw, hw,
                                                   stream), "pww_sampler_update_rescale")

    def graph_of(fn):
        s = torch.cuda.Stream(device=device)
        with torch.cuda.stream(s):
            for _ in range(3):
                fn()
        s.synchronize()
        graph = torch.cuda.CUDAGraph()
        with torch.cuda.graph(graph, stream=s):
            for _ in range(iters):
                fn()
        return graph

    graphs = {"plain": graph_of(plain), "rescale": graph_of(rescale)}
    times = {k: [] for k in graphs}
    for _ in range(reps):                                       # alternated
        for k, gr in graphs.items():
            lat.normal_().mul_(14.6)                            # keep the latents finite over the rounds
            hist.zero_()
            times[k].append(_events_ms(gr.replay) * 1e3 / iters)
    return {f"{k}_us": float(np.median(v)) for k, v in times.items()}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=30)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--no-loop", action="store_true")
    ap.add_argument("--no-update", action="store_true")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_vpred.py needs a CUDA device (H100)")
    device = torch.device("cuda", 0)
    torch.cuda.set_device(device)
    torch.backends.cudnn.benchmark = True
    line = {"metric": "vpred_guidance_rescale_steps_per_sec_768sq", "unit": "steps/s, us per launch",
            "config": {"workload": f"synthetic:sd21 {SIZE}x{SIZE}, aurora map, LMS v_prediction, {args.steps} steps, "
                                   "fp16, CFG 7.5, CUDA graph", "phis": list(PHIS), "reps": args.reps},
            "device": bench.device_info(0)}
    with torch.no_grad():
        if not args.no_loop:
            line["loop"] = loop(device, args.steps, args.reps)
        if not args.no_update:
            line["update"] = {f"m{m}_{hw}x{hw}": update(device, m, hw) for m in (1, 8) for hw in (64, 96)}
    print(json.dumps(line), flush=True)


if __name__ == "__main__":
    main()
