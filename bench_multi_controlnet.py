#!/usr/bin/env python
"""bench_multi_controlnet.py -- the default workload with 0 to 3 ControlNets, and the multi-ControlNet combine launch.

    python bench_multi_controlnet.py [--rounds 3] [--no-loop] [--no-kernel]

Loop: bench.py's default workload (aurora_1 map, SD1.5-shaped fp16 UNet, 512x512, 30 LMS steps, CFG 7.5, CUDA graph,
one image per sampler) in five cases that alternate for --rounds rounds: no ControlNet; 1, 2 and 3 SD1.5-shaped
ControlNets of seeds 1, 2, 3 over the whole run; 2 ControlNets in the disjoint windows [0, 0.5] and [0.5, 1].  Each run
is timed whole after a warm-up pass (graph capture) with CUDA events; every case reports the median steps/s and
images/s, the range, the native launches per step of each active set's graph, the SM clock nvidia-smi sampled during
each window, and the memory it added: `torch.cuda.max_memory_allocated` over its set-up and warm-up (one graph pool per
active set) above what was allocated before it.

Kernel: one pww_control_combine_f16 launch over the 13 SD1.5 residuals at 512x512 (rows = 2m) of U = 2 and 3 units,
m = 1 and 8, against the torch ops it replaces (per level U `mul` and U - 1 `add`), microseconds from CUDA events
around a CUDA graph of back-to-back calls, and the kernel's GB/s.

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
from bench_controlnet import _hint  # noqa: E402
from bench_dtype import _events_ms  # noqa: E402
from paint_with_words_sd_b200 import fused_ops  # noqa: E402
from paint_with_words_sd_b200.conditioning import _encode_text_color_inputs  # noqa: E402
from paint_with_words_sd_b200.controlnet import build_controlnet, residual_shapes  # noqa: E402
from paint_with_words_sd_b200.scheduler import LMSDiscreteScheduler  # noqa: E402
from paint_with_words_sd_b200.synthetic import RandomTextEncoder, SimpleWordTokenizer  # noqa: E402
from paint_with_words_sd_b200.unet import build_unet  # noqa: E402
from tests.fixtures import SETTINGS, color_map_image  # noqa: E402

STEPS = 30
# case -> (number of ControlNets, extra PwWSampler arguments)
CASES = {"plain": (0, {}), "controlnets_1": (1, {}), "controlnets_2": (2, {}), "controlnets_3": (3, {}),
         "controlnets_2_disjoint": (2, {"control_guidance_start": [0.0, 0.5], "control_guidance_end": [0.5, 1.0]})}


def _hints(size: int, k: int):
    """k different scribble-like hints: bench_controlnet's, rolled."""
    h = _hint(size)
    return [torch.roll(h, shifts=(size // 5 * u, size // 7 * u), dims=(2, 3)) for u in range(k)]


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
    runs, memory = {}, {}
    try:
        unet = build_unet(ucfg, seed=0, dtype=torch.float16, device=device)
        nets = [build_controlnet(ucfg, seed=1 + u, dtype=torch.float16, device=device) for u in range(3)]
        P.patch_unet(unet)
        for net in nets:
            P.patch_unet(net)
        for name, (k, kw) in CASES.items():
            torch.cuda.synchronize(device)
            base = torch.cuda.memory_allocated(device)
            torch.cuda.reset_peak_memory_stats(device)
            sch = LMSDiscreteScheduler(beta_start=0.00085, beta_end=0.012, beta_schedule="scaled_linear")
            sch.set_timesteps(STEPS)
            lat = (lat0 * sch.init_noise_sigma).to(device)
            control = {} if k == 0 else dict(controlnet=nets[:k], control_image=_hints(size, k), **kw)
            smp = PwWSampler(unet, sch, [cond], [uncond], lat, bench.weight_function, bench.GUIDANCE, **control)

            def run(smp=smp, lat=lat):
                smp.restart(lat)
                for _ in range(STEPS):
                    smp.step()
            run()                                               # warm-up: graph capture, library autotune
            torch.cuda.synchronize(device)
            memory[name] = {"base_bytes": base, "max_allocated_bytes": torch.cuda.max_memory_allocated(device),
                            "added_bytes": torch.cuda.max_memory_allocated(device) - base}
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
                     "native_launches_per_active_set": {"".join("1" if a else "0" for a in key) or "plain": n
                                                        for key, n in smp.native_launches_per_active_set.items()},
                     "steps_per_active_set": {"".join("1" if a else "0" for a in key) or "plain":
                                              smp._active_sets.count(key) for key in set(smp._active_sets)},
                     "memory": memory[name],
                     "sm_mhz": [c["sm_mhz"] for c in clocks[name]],
                     "clock_reasons": sorted({r for c in clocks[name] for r in c["reasons"]})}
    return res


def combine_us(device, units: int, m: int, iters=64, reps=5, target_mb=192) -> dict:
    """Microseconds per combine of `units` sets of the 13 SD1.5 residuals (rows = 2m) at 512x512: one
    pww_control_combine_f16 launch against the per-level torch ops, both over back-to-back calls cycling through more
    than L2 of buffers."""
    shapes = residual_shapes(bench.unet_config(bench.CONFIGS[2]["unet"]), bench.CONFIGS[2]["size"] // 8)
    rows = 2 * m
    elems = sum(rows * c * h * w for c, h, w in shapes)
    per_set = elems * 2 * (units + 1)
    nsets = max(2, int(np.ceil(target_mb * 1e6 / per_set)))
    g = torch.Generator().manual_seed(0)

    def cl(t):
        return t.to(device, torch.float16).contiguous(memory_format=torch.channels_last)
    sets = [([[cl(torch.randn(rows, *s, generator=g)) for s in shapes] for _ in range(units)],
             [cl(torch.empty(rows, *s)) for s in shapes]) for _ in range(nsets)]
    scales = torch.rand(units, len(shapes), rows, generator=g).to(device)
    cols = [[scales[u, k].view(rows, 1, 1, 1).half() for k in range(len(shapes))] for u in range(units)]

    def native(i):
        res, out = sets[i % nsets]
        fused_ops.control_combine(res, scales, out)

    def torch_ops(i):
        res, out = sets[i % nsets]
        for k, o in enumerate(out):
            torch.mul(res[0][k], cols[0][k], out=o)
            for u in range(1, units):
                o.add_(res[u][k].mul(cols[u][k]))

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
    out["bytes_per_launch"] = int(elems * 2 * (units + 1))          # read every unit's residuals, write the sum
    out["native_GB_per_s"] = out["bytes_per_launch"] / (out["native_us"] * 1e3)
    out["torch_GB_per_s_equivalent"] = out["bytes_per_launch"] / (out["torch_us"] * 1e3)
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--no-loop", action="store_true")
    ap.add_argument("--no-kernel", action="store_true")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_multi_controlnet.py needs a CUDA device (H100)")
    device = torch.device("cuda", 0)
    torch.cuda.set_device(device)
    torch.backends.cudnn.benchmark = True
    line = {"metric": "multi_controlnet_steps_per_sec_512sq_cfg", "unit": "steps/s, images/s, us, bytes",
            "config": {"workload": bench.CONFIGS[2]["what"], "steps": STEPS, "cuda_graph": True, "rounds": args.rounds,
                       "controlnets": "SD1.5-shaped, seeded random weights (seeds 1, 2, 3), fp16",
                       "kernel": "pww_control_combine_f16 over the 13 SD1.5 residuals at 512x512, rows = 2m"},
            "device": bench.device_info(0)}
    with torch.no_grad():
        if not args.no_loop:
            line["loop"] = loop(device, args.rounds)
        if not args.no_kernel:
            line["kernel"] = {f"U{u}_m{m}": combine_us(device, u, m) for u in (2, 3) for m in (1, 8)}
    print(json.dumps(line), flush=True)


if __name__ == "__main__":
    main()
