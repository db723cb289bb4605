#!/usr/bin/env python
"""bench_samplers.py -- the samplers on the default workload, and the native step tail against the torch one it replaced.

    python bench_samplers.py [--samplers lms,euler,euler_a,dpmpp_2m_karras] [--ms 1,8] [--reps 3] [--no-loop] [--no-tail]

Loop: bench.py's default workload (aurora_1 map, SD1.5-shaped UNet, 512x512, fp16, CFG 7.5, CUDA graph) with LMS at 30
steps, Euler at 30, Euler ancestral at 30 and DPM++ 2M with Karras sigmas at 20, m images per sampler.  Each schedule is
timed whole after a warm-up pass (graph capture) with CUDA events; the samplers are run interleaved, --reps rounds, and
each gets the median, the range, and the SM clock nvidia-smi sampled during each of its windows: steps/s counts one
denoising step of one image, images/s finished images.  Fewer steps per image are only worth it if the images hold up, which
synthetic weights cannot show.

Tail: the step around the UNet at 64x64 latents, fp16 channels-last eps, m images, LMS coefficients: the previous
release's torch ops (scale, two cats, fp16 cast, .float(), CFG, roll, two copies, multiply, sum, add) against
pww_sampler_input + pww_sampler_update; microseconds per step from CUDA events over a CUDA graph of back-to-back steps,
and kernels per step counted with torch.profiler.

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

import bench  # noqa: E402  (workload definition, device info)
from paint_with_words_sd_b200 import _native  # noqa: E402
from paint_with_words_sd_b200.conditioning import _encode_text_color_inputs  # noqa: E402
from paint_with_words_sd_b200.scheduler import (DPMSolverMultistepScheduler, EulerAncestralDiscreteScheduler,  # noqa: E402
                                                EulerDiscreteScheduler, LMSDiscreteScheduler)
from paint_with_words_sd_b200.synthetic import RandomTextEncoder, SimpleWordTokenizer  # noqa: E402
from paint_with_words_sd_b200.unet import build_unet  # noqa: E402
from tests.fixtures import SETTINGS, color_map_image  # noqa: E402

SAMPLERS = (("lms", LMSDiscreteScheduler, 30), ("euler", EulerDiscreteScheduler, 30),
            ("euler_a", EulerAncestralDiscreteScheduler, 30),
            ("dpmpp_2m_karras", functools.partial(DPMSolverMultistepScheduler, use_karras_sigmas=True), 20))
KW = dict(beta_start=0.00085, beta_end=0.012, beta_schedule="scaled_linear")


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


def loop(device, names, ms, reps: int) -> dict:
    import paint_with_words_sd_b200 as P
    from paint_with_words_sd_b200.pipeline import PwWSampler, initial_latents
    cfg = bench.CONFIGS[2]
    size = cfg["size"]
    unet = build_unet(bench.unet_config(cfg["unet"]), seed=0, dtype=torch.float16, device=device)
    unet = unet.to(memory_format=torch.channels_last)
    P.patch_unet(unet)
    res = {}
    try:
        tok, enc = SimpleWordTokenizer(), RandomTextEncoder(cfg["text_dim"]).to(device)
        s = SETTINGS["aurora"]
        images = []
        for i in range(max(ms)):
            seeds, sep, cond, uncond = _encode_text_color_inputs(enc, tok, device, color_map_image("aurora", size),
                                                                 dict(s["ctx"]), s["prompt"], "")
            images.append((cond, uncond, initial_latents((1, 4, size // 8, size // 8), i, seeds, sep)))
        chosen = [x for x in SAMPLERS if x[0] in names]
        with torch.no_grad():
            for m in ms:
                part = images[:m]
                runs = []
                for name, cls, steps in chosen:
                    sch = cls(**KW)
                    sch.set_timesteps(steps)
                    lat = (torch.cat([x[2] for x in part], 0) * sch.init_noise_sigma).to(device)
                    smp = PwWSampler(unet, sch, [x[0] for x in part], [x[1] for x in part], lat, bench.weight_function,
                                     bench.GUIDANCE, noise_seed=list(range(m)))
                    run = functools.partial(_full_run, smp, lat, steps)
                    run()                                           # warm-up: graph capture, library autotune
                    runs.append((name, steps, smp, run))
                times = {name: [] for name, _, _, _ in runs}
                clocks = {name: [] for name, _, _, _ in runs}
                for _ in range(reps):                               # interleaved: drift of the card hits every sampler
                    for name, _, _, run in runs:
                        with bench.ClockSampler(device.index or 0) as clk:
                            times[name].append(_events_ms(run))
                        clocks[name].append(clk.summary())
                for name, steps, smp, _ in runs:
                    t = float(np.median(times[name]))
                    res[f"{name}_{steps}_m{m}"] = {
                        "steps_per_s": m * steps / (t / 1e3), "images_per_s": m / (t / 1e3),
                        "steps_per_s_range": [m * steps / (max(times[name]) / 1e3), m * steps / (min(times[name]) / 1e3)],
                        "ms_per_image_batch": t, "native_launches_per_step": smp.native_launches_per_step,
                        "sm_mhz": [c["sm_mhz"] for c in clocks[name]],
                        "clock_reasons": sorted({r for c in clocks[name] for r in c["reasons"]})}
                del runs
                torch.cuda.empty_cache()
    finally:
        P.unpatch_all()
    return res


def tail(device, m: int, iters: int = 200, reps: int = 5) -> dict:
    h = w = 64
    L = _native.lib()
    g = torch.Generator().manual_seed(0)
    lat = (torch.randn(m, 4, h, w, generator=g) * 14.6).to(device)
    eps = torch.randn(2 * m, 4, h, w, generator=g).half().to(device).contiguous(memory_format=torch.channels_last)
    params = torch.tensor([14.6, 1 / (14.6 ** 2 + 1) ** 0.5, 999.0, 0.5, -0.2, 0.1, -0.05, 7.5, 0.0, 1.0, 0.0, 1.0,
                           0.0, 0.0, 0.0], device=device)
    gscale = torch.full((m, 1, 1, 1), 7.5, device=device)
    derivs = torch.zeros(4, m, 4, h, w, device=device)
    unet_in = torch.empty(2 * m, 4, h, w, dtype=torch.float16, device=device)
    form = params.data_ptr() + 9 * 4

    def torch_tail():
        x = lat * params[1]
        x2 = torch.cat([x, x], 0).to(torch.float16)
        e = eps.float()
        noise_pred = e[m:] + gscale * (e[:m] - e[m:])
        derivs.copy_(torch.roll(derivs, 1, 0))
        derivs[0].copy_(noise_pred)
        lat.add_((params[3:7].view(4, 1, 1, 1, 1) * derivs).sum(0))
        return x2

    def native_tail():
        stream = torch.cuda.current_stream(device).cuda_stream
        _native.check(L.pww_sampler_input(lat.data_ptr(), params.data_ptr() + 4, None, unet_in.data_ptr(),
                                          _native.PWW_DTYPE_F16, m, 4, h, w, stream), "pww_sampler_input")
        _native.check(L.pww_sampler_update(eps.data_ptr(), _native.PWW_DTYPE_F16, *eps.stride(), lat.data_ptr(),
                                           derivs.data_ptr(), 4, None, gscale.data_ptr(), params.data_ptr() + 12,
                                           form, m, h, w, stream), "pww_sampler_update")

    def timed(fn):
        s = torch.cuda.Stream(device=device)
        with torch.cuda.stream(s):
            for _ in range(3):
                fn()
        s.synchronize()
        graph = torch.cuda.CUDAGraph()
        with torch.cuda.graph(graph, stream=s):
            for _ in range(iters):
                fn()
        return float(np.median([_events_ms(graph.replay) * 1e3 / iters for _ in range(reps)]))

    def kernels(fn):
        from torch.profiler import ProfilerActivity, profile
        torch.cuda.synchronize()
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            fn()
            torch.cuda.synchronize()
        return sum(1 for e in prof.events() if e.device_type.name == "CUDA")

    return {"torch_us": timed(torch_tail), "native_us": timed(native_tail),
            "torch_kernels_per_step": kernels(torch_tail), "native_kernels_per_step": kernels(native_tail)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--samplers", default=",".join(n for n, _, _ in SAMPLERS),
                    help="which samplers to time")
    ap.add_argument("--ms", default="1,8", help="images per sampler")
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--no-loop", action="store_true")
    ap.add_argument("--no-tail", action="store_true")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_samplers.py needs a CUDA device (H100)")
    ms = [int(x) for x in args.ms.split(",")]
    device = torch.device("cuda", 0)
    torch.cuda.set_device(device)
    torch.backends.cudnn.benchmark = True
    line = {"metric": "sampler_steps_and_images_per_sec_512sq_cfg", "unit": "steps/s, images/s",
            "config": {"workload": bench.CONFIGS[2]["what"], "samplers": [f"{n}@{k}" for n, _, k in SAMPLERS],
                       "cuda_graph": True, "reps": args.reps},
            "device": bench.device_info(0)}
    with torch.no_grad():
        if not args.no_loop:
            line["loop"] = loop(device, args.samplers.split(","), ms, args.reps)
        if not args.no_tail:                   # last: the profiler it uses for kernel counts slows later launches
            line["tail"] = {f"m{m}": tail(device, m) for m in ms}
    print(json.dumps(line), flush=True)


if __name__ == "__main__":
    main()
