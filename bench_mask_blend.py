#!/usr/bin/env python
"""bench_mask_blend.py -- what masked img2img costs: the default workload as img2img with and without a mask, and the
sampler update launch alone, unmasked against masked.

    python bench_mask_blend.py [--reps 5] [--steps 30] [--strength 0.75] [--no-loop] [--no-update]

Loop: the SD1.5-shaped UNet (synthetic:sd15, seeded random weights) at 512x512 (64x64 latents), the aurora colour map,
one image, LMS, fp16, CFG 7.5, CUDA-graph replay, img2img at strength 0.75 of 30 steps (the last 22): seeded init
latents noised to the first step's sigma.  Two samplers, one unmasked (pww_sampler_update) and one with the right half
of the frame masked for repainting (pww_sampler_update_masked), are timed whole with CUDA events after a warm-up run
(graph capture), alternated over --reps rounds; each gets the median and the range of steps/s.

Update: the update launch alone at 64x64 and 96x96 latents, m = 1 and 8, fp16 channels-last UNet output, an LMS step
form with a full history ring: microseconds per launch from CUDA events over a CUDA graph of 200 back-to-back launches,
alternated: plain against masked, and rescale (phi 0.7) against masked + rescale.

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

KW = dict(beta_start=0.00085, beta_end=0.012, beta_schedule="scaled_linear")
SIZE = 512
MODES = ("unmasked", "masked")


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


def loop(device, steps: int, strength: float, reps: int) -> dict:
    import paint_with_words_sd_b200 as P
    from paint_with_words_sd_b200.pipeline import PwWSampler
    cfg = UNetConfig.sd15()
    unet = build_unet(cfg, seed=0, dtype=torch.float16, device=device).to(memory_format=torch.channels_last)
    P.patch_unet(unet)
    h = w = SIZE // 8
    try:
        tok, enc = SimpleWordTokenizer(), RandomTextEncoder(cfg.cross_attention_dim).to(device)
        s = SETTINGS["aurora"]
        _, _, cond, uncond = _encode_text_color_inputs(enc, tok, device, color_map_image("aurora", SIZE),
                                                       dict(s["ctx"]), s["prompt"], "")
        g = torch.Generator().manual_seed(0)
        init = torch.randn(1, 4, h, w, generator=g).to(device)
        noise = torch.randn(1, 4, h, w, generator=g).to(device)
        mask = torch.zeros(1, 1, h, w, device=device)
        mask[..., w // 2:] = 1
        runs = {}
        for mode in MODES:
            sch = LMSDiscreteScheduler(**KW)
            sch.set_timesteps(steps)
            ts = sch.timesteps[steps - min(int(steps * strength), steps):]
            lat = sch.add_noise(init, noise, ts[:1])
            blend = dict(init_latents=init, init_noise=noise, inpaint_mask=mask) if mode == "masked" else {}
            smp = PwWSampler(unet, sch, [cond], [uncond], lat, bench.weight_function, 7.5, timesteps=ts, **blend)
            run = functools.partial(_full_run, smp, lat, len(ts))
            run()                                               # warm-up: graph capture, library autotune
            runs[mode] = (smp, run, len(ts))
        times = {mode: [] for mode in MODES}
        for _ in range(reps):                                   # alternated: drift of the card hits both
            for mode in MODES:
                times[mode].append(_events_ms(runs[mode][1]))
        res = {}
        for mode in MODES:
            t, n = times[mode], runs[mode][2]
            smp = runs[mode][0]
            res[mode] = {"steps_per_s": n / (float(np.median(t)) / 1e3),
                         "steps_per_s_range": [n / (max(t) / 1e3), n / (min(t) / 1e3)],
                         "ms_per_run": float(np.median(t)), "steps": n,
                         "native_launches_per_step": smp.native_launches_per_step,
                         "finite": bool(torch.isfinite(smp.latents).all())}
        kept = runs["masked"][0].latents[..., : w // 2]
        res["masked"]["kept_area_equals_init"] = bool(torch.equal(kept, init[..., : w // 2]))
        return res
    finally:
        P.unpatch_all()


def update(device, m: int, hw: int, iters: int = 200, reps: int = 5) -> dict:
    L = _native.lib()
    g = torch.Generator().manual_seed(0)
    lat = (torch.randn(m, 4, hw, hw, generator=g) * 14.6).to(device)
    eps = torch.randn(2 * m, 4, hw, hw, generator=g).half().to(device).contiguous(memory_format=torch.channels_last)
    init = torch.randn(m, 4, hw, hw, generator=g).to(device)
    noise0 = torch.randn(m, 4, hw, hw, generator=g).to(device)
    mask = torch.zeros(m, 1, hw, hw, device=device)
    mask[..., hw // 2:] = 1
    sigma_next = torch.tensor([13.9], device=device)
    gscale = torch.full((m,), 7.5, device=device)
    phi = torch.full((m,), 0.7, device=device)
    beta = torch.tensor([0.5, -0.2, 0.1, -0.05], device=device)
    form = torch.tensor([1.0, 0.0, 1.0, 0.0, 0.0, 0.0], device=device)      # LMS: q = eps
    hist = torch.zeros(4, m, 4, hw, hw, device=device)

    def launch(rescale: bool, masked: bool):
        stream = torch.cuda.current_stream(device).cuda_stream
        args = (eps.data_ptr(), _native.PWW_DTYPE_F16, *eps.stride(), lat.data_ptr(), hist.data_ptr(), 4, None,
                gscale.data_ptr(), beta.data_ptr(), form.data_ptr())
        if masked:
            _native.check(L.pww_sampler_update_masked(*args, phi.data_ptr() if rescale else None, None,
                                                      init.data_ptr(), noise0.data_ptr(), mask.data_ptr(),
                                                      sigma_next.data_ptr(), m, hw, hw, stream),
                          "pww_sampler_update_masked")
        elif rescale:
            _native.check(L.pww_sampler_update_rescale(*args, phi.data_ptr(), None, m, hw, hw, stream),
                          "pww_sampler_update_rescale")
        else:
            _native.check(L.pww_sampler_update(*args, m, hw, hw, stream), "pww_sampler_update")

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

    kinds = {"plain": (False, False), "masked": (False, True), "rescale": (True, False),
             "masked_rescale": (True, True)}
    graphs = {k: graph_of(functools.partial(launch, *v)) for k, v in kinds.items()}
    times = {k: [] for k in graphs}
    for _ in range(reps):                                       # alternated
        for k, gr in graphs.items():
            lat.normal_().mul_(14.6)                            # keep the latents finite over the rounds
            hist.zero_()
            times[k].append(_events_ms(gr.replay) * 1e3 / iters)
    # the extra reads of a masked launch: init, noise0 (4 fp32 each) and the mask (1 fp32) per pixel and image
    extra = m * hw * hw * 9 * 4
    return {**{f"{k}_us": float(np.median(v)) for k, v in times.items()}, "masked_extra_bytes": extra}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=30)
    ap.add_argument("--strength", type=float, default=0.75)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--no-loop", action="store_true")
    ap.add_argument("--no-update", action="store_true")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_mask_blend.py needs a CUDA device (H100)")
    device = torch.device("cuda", 0)
    torch.cuda.set_device(device)
    torch.backends.cudnn.benchmark = True
    line = {"metric": "mask_blend_img2img_steps_per_sec_512sq", "unit": "steps/s, us per launch",
            "config": {"workload": f"synthetic:sd15 {SIZE}x{SIZE}, aurora map, LMS, img2img strength {args.strength} "
                                   f"of {args.steps} steps, fp16, CFG 7.5, CUDA graph; mask: right half",
                       "reps": args.reps},
            "device": bench.device_info(0)}
    with torch.no_grad():
        if not args.no_loop:
            line["loop"] = loop(device, args.steps, args.strength, args.reps)
        if not args.no_update:
            line["update"] = {f"m{m}_{hw}x{hw}": update(device, m, hw) for m in (1, 8) for hw in (64, 96)}
    print(json.dumps(line), flush=True)


if __name__ == "__main__":
    main()
