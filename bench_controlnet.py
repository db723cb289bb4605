#!/usr/bin/env python
"""bench_controlnet.py -- the default workload with and without a ControlNet, and the residual-injection launch.

    python bench_controlnet.py [--rounds 3] [--no-loop] [--no-kernel]

Loop: bench.py's default workload (aurora_1 map, SD1.5-shaped fp16 UNet, 512x512, 30 LMS steps, CFG 7.5, CUDA graph,
one image per sampler) in four cases that alternate for --rounds rounds: no ControlNet; an SD1.5-shaped ControlNet;
the same in guess mode; the same with the guidance window [0, 0.5].  Each run is timed whole after a warm-up pass
(graph capture) with CUDA events; every case reports the median steps/s and images/s, the range, the native launches
per step of its graphs and the SM clock nvidia-smi sampled during each window.

Kernel: one pww_control_inject_f16 launch over the 13 SD1.5 residuals at 512x512 (rows = 2m, m = 1 and 8) against the
13 `mul` + 13 `add` torch ops it replaces, microseconds from CUDA events around a CUDA graph of back-to-back calls.

One JSON line on stdout, with the GPU's name, power limit and SM clock.  Writes nothing.
"""
from __future__ import annotations

import argparse
import json
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, ROOT)

import bench  # noqa: E402  (workload definition, device info, clock sampler)
from bench_dtype import _events_ms  # noqa: E402
from paint_with_words_sd_b200 import fused_ops  # noqa: E402
from paint_with_words_sd_b200.conditioning import _encode_text_color_inputs  # noqa: E402
from paint_with_words_sd_b200.controlnet import build_controlnet, residual_shapes  # noqa: E402
from paint_with_words_sd_b200.scheduler import LMSDiscreteScheduler  # noqa: E402
from paint_with_words_sd_b200.synthetic import RandomTextEncoder, SimpleWordTokenizer  # noqa: E402
from paint_with_words_sd_b200.unet import build_unet  # noqa: E402
from tests.fixtures import SETTINGS, color_map_image  # noqa: E402

STEPS = 30
CASES = {"plain": None, "controlnet": {}, "guess_mode": {"guess_mode": True},
         "window_0_0.5": {"control_guidance_start": 0.0, "control_guidance_end": 0.5}}


def _hint(size: int) -> torch.Tensor:
    """A scribble-like [1, 3, size, size] hint in [0, 1]."""
    g = torch.Generator().manual_seed(7)
    img = torch.zeros(1, 3, size, size)
    for _ in range(12):
        y, x = torch.randint(0, size - size // 4, (2,), generator=g).tolist()
        img[:, :, y:y + size // 8, x:x + size // 4] = torch.rand(3, 1, 1, generator=g)
    return img


def loop(device, rounds: int) -> dict:
    import paint_with_words_sd_b200 as P
    from paint_with_words_sd_b200.pipeline import PwWSampler, initial_latents
    cfg = bench.CONFIGS[2]
    size = cfg["size"]
    ucfg = bench.unet_config(cfg["unet"])
    tok, enc = SimpleWordTokenizer(), RandomTextEncoder(cfg["text_dim"]).to(device)
    s = SETTINGS["aurora"]
    seeds, sep, cond, uncond = _encode_text_color_inputs(enc, tok, device, color_map_image("aurora", size),
                                                         dict(s["ctx"]), s["prompt"], "")
    lat0 = initial_latents((1, 4, size // 8, size // 8), 0, seeds, sep)
    runs = {}
    try:
        unet = build_unet(ucfg, seed=0, dtype=torch.float16, device=device)
        net = build_controlnet(ucfg, seed=1, dtype=torch.float16, device=device)
        P.patch_unet(unet)
        P.patch_unet(net)
        for name, kw in CASES.items():
            sch = LMSDiscreteScheduler(beta_start=0.00085, beta_end=0.012, beta_schedule="scaled_linear")
            sch.set_timesteps(STEPS)
            lat = (lat0 * sch.init_noise_sigma).to(device)
            control = {} if kw is None else dict(controlnet=net, control_image=_hint(size), **kw)
            smp = PwWSampler(unet, sch, [cond], [uncond], lat, bench.weight_function, bench.GUIDANCE, **control)

            def run(smp=smp, lat=lat):
                smp.restart(lat)
                for _ in range(STEPS):
                    smp.step()
            run()                                               # warm-up: graph capture, library autotune
            runs[name] = (smp, run)
        times = {n: [] for n in CASES}
        clocks = {n: [] for n in CASES}
        for _ in range(rounds):                                 # alternating: drift of the card hits every case
            for name in CASES:
                with bench.ClockSampler(device.index or 0) as clk:
                    times[name].append(_events_ms(runs[name][1]))
                clocks[name].append(clk.summary())
    finally:
        P.unpatch_all()
    res = {}
    for name in CASES:
        t = times[name]
        smp = runs[name][0]
        res[name] = {"steps_per_s": STEPS / (float(np.median(t)) / 1e3),
                     "images_per_s": 1.0 / (float(np.median(t)) / 1e3),
                     "steps_per_s_range": [STEPS / (max(t) / 1e3), STEPS / (min(t) / 1e3)],
                     "native_launches_per_step": smp.native_launches_per_step,
                     "native_launches_per_step_without_control": smp.native_launches_per_step_without_control,
                     "sm_mhz": [c["sm_mhz"] for c in clocks[name]],
                     "clock_reasons": sorted({r for c in clocks[name] for r in c["reasons"]})}
    return res


def inject_us(device, m: int, iters=64, reps=5, target_mb=192) -> dict:
    """Microseconds per injection of the 13 SD1.5 residuals (rows = 2m) at 512x512: one pww_control_inject_f16 launch
    against the 13 mul + 13 add torch ops, both over back-to-back calls cycling through more than L2 of buffers."""
    shapes = residual_shapes(bench.unet_config(bench.CONFIGS[2]["unet"]), bench.CONFIGS[2]["size"] // 8)
    B = 2 * m
    per_set = sum(B * c * h * w * 2 * 2 for c, h, w in shapes)
    nsets = max(2, int(np.ceil(target_mb * 1e6 / per_set)))
    g = torch.Generator().manual_seed(0)

    def cl(t):
        return t.to(device, torch.float16).contiguous(memory_format=torch.channels_last)
    sets = [([cl(torch.randn(B, *s, generator=g)) for s in shapes], [cl(torch.randn(B, *s, generator=g)) for s in shapes])
            for _ in range(nsets)]
    scales = torch.rand(len(shapes), B, generator=g).to(device)
    col = [scales[k].view(B, 1, 1, 1).half() for k in range(len(shapes))]      # fp16: one mul, one add per level

    def native(i):
        dst, res = sets[i % nsets]
        fused_ops.control_inject(dst, res, scales)

    def torch_ops(i):
        dst, res = sets[i % nsets]
        for k, (d, r) in enumerate(zip(dst, res)):
            d.add_(r.mul(col[k]))

    out = {}
    for name, fn in (("native_us", native), ("torch_us", torch_ops)):
        s = torch.cuda.Stream(device=device)
        with torch.cuda.stream(s):
            for i in range(3):
                fn(i)
        s.synchronize()
        graph = torch.cuda.CUDAGraph()
        with torch.cuda.graph(graph, stream=s):
            for i in range(iters):
                fn(i)
        out[name] = float(np.median([_events_ms(graph.replay) * 1e3 / iters for _ in range(reps)]))
    out["bytes_per_launch"] = int(sum(B * c * h * w * 2 * 3 for c, h, w in shapes))   # read dst + res, write dst
    out["native_GB_per_s"] = out["bytes_per_launch"] / (out["native_us"] * 1e3)
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--no-loop", action="store_true")
    ap.add_argument("--no-kernel", action="store_true")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_controlnet.py needs a CUDA device (H100)")
    device = torch.device("cuda", 0)
    torch.cuda.set_device(device)
    torch.backends.cudnn.benchmark = True
    line = {"metric": "controlnet_steps_per_sec_512sq_cfg", "unit": "steps/s, images/s, us",
            "config": {"workload": bench.CONFIGS[2]["what"], "steps": STEPS, "cuda_graph": True, "rounds": args.rounds,
                       "controlnet": "SD1.5-shaped, seeded random weights, fp16",
                       "kernel": "pww_control_inject_f16 over the 13 SD1.5 residuals at 512x512, rows = 2m"},
            "device": bench.device_info(0)}
    with torch.no_grad():
        if not args.no_loop:
            line["loop"] = loop(device, args.rounds)
        if not args.no_kernel:
            line["kernel"] = {f"m{m}": inject_us(device, m) for m in (1, 8)}
    print(json.dumps(line), flush=True)


if __name__ == "__main__":
    main()
