#!/usr/bin/env python
"""bench_t2i_adapter.py -- the default workload with T2I-Adapter units, and the fused adapter-residual launch.

    python bench_t2i_adapter.py [--rounds 3] [--no-loop] [--no-kernel]

Loop: bench.py's default workload (aurora_1 map, SD1.5-shaped fp16 UNet, 512x512, 30 LMS steps, CFG 7.5, CUDA graph,
one image per sampler) in five cases that alternate for --rounds rounds: no control unit; one full adapter (the image /
keypose shape: cin 192, nums_rb 2); one light adapter (the color shape); a full adapter + an SD1.5-shaped ControlNet;
the ControlNet alone.  Each run is timed whole after a warm-up pass (graph capture) with CUDA events; every case reports
the median steps/s, the range, the native launches of each active set's graph, the SM clock sampled during each window
and, for adapter cases, the one-time set-up cost (the sampler's construction, which runs the adapter once).

Kernel: one pww_adapter_residual_f16 launch at each SD1.5 512x512 encoder-level shape (rows = 2m, feature on every
row, m = 1 and 8), against torch's `proj + res` alone (what a plain step runs there) and `proj + res` followed by a
separate `+ feat` (what the adapter would cost without the fusion).  Microseconds from CUDA events around a CUDA graph of
back-to-back calls cycling through more than L2 of buffers; the share of the 3.35 TB/s HBM3 bound is the bytes the
fused launch must move (read a, b, feat; write out) over its time.

One JSON line on stdout, with the GPU's name, power limit and SM clock.  Writes nothing.
"""
from __future__ import annotations

import argparse
import json
import os
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, ROOT)

import bench  # noqa: E402  (workload definition, device info, clock sampler)
from bench_controlnet import _hint  # noqa: E402
from bench_dtype import _events_ms  # noqa: E402
from paint_with_words_sd_b200 import fused_ops  # noqa: E402
from paint_with_words_sd_b200.adapter import build_adapter, unet_level_sizes  # noqa: E402
from paint_with_words_sd_b200.conditioning import _encode_text_color_inputs  # noqa: E402
from paint_with_words_sd_b200.controlnet import build_controlnet  # noqa: E402
from paint_with_words_sd_b200.scheduler import LMSDiscreteScheduler  # noqa: E402
from paint_with_words_sd_b200.synthetic import RandomTextEncoder, SimpleWordTokenizer  # noqa: E402
from paint_with_words_sd_b200.unet import build_unet  # noqa: E402
from tests.fixtures import SETTINGS, color_map_image  # noqa: E402

STEPS = 30
HBM_BYTES_PER_S = 3.35e12        # H100 SXM data sheet
CASES = ("plain", "full_adapter", "light_adapter", "adapter_controlnet", "controlnet")


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
    runs, setup_ms = {}, {}
    try:
        unet = build_unet(ucfg, seed=0, dtype=torch.float16, device=device)
        net = build_controlnet(ucfg, seed=1, dtype=torch.float16, device=device)
        full = build_adapter(ucfg, "full", 192, seed=3, dtype=torch.float16, device=device)
        light = build_adapter(ucfg, "light", 192, seed=4, dtype=torch.float16, device=device)
        P.patch_unet(unet)
        P.patch_unet(net)
        units = {"plain": [], "full_adapter": [full], "light_adapter": [light], "adapter_controlnet": [full, net],
                 "controlnet": [net]}
        for name in CASES:
            sch = LMSDiscreteScheduler(beta_start=0.00085, beta_end=0.012, beta_schedule="scaled_linear")
            sch.set_timesteps(STEPS)
            lat = (lat0 * sch.init_noise_sigma).to(device)
            u = units[name]
            control = dict(controlnet=u, control_image=[_hint(size)] * len(u)) if u else {}
            for _ in range(2):          # the second construction is timed: the first loads modules and autotunes
                torch.cuda.synchronize()
                t0 = time.perf_counter()
                smp = PwWSampler(unet, sch, [cond], [uncond], lat, bench.weight_function, bench.GUIDANCE, **control)
                torch.cuda.synchronize()
                setup_ms[name] = (time.perf_counter() - t0) * 1e3

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
                     "steps_per_s_range": [STEPS / (max(t) / 1e3), STEPS / (min(t) / 1e3)],
                     "native_launches_per_active_set": {str(k): v for k, v in
                                                        smp.native_launches_per_active_set.items()},
                     "sampler_setup_ms": setup_ms[name],
                     "sm_mhz": [c["sm_mhz"] for c in clocks[name]],
                     "clock_reasons": sorted({r for c in clocks[name] for r in c["reasons"]})}
    return res


def level_us(device, C: int, h: int, w: int, m: int, iters=64, reps=5, target_mb=192) -> dict:
    """Microseconds per call at one level shape [2m, C, h, w] fp16 channels-last: the fused launch, torch's `proj + res`,
    and `proj + res` then `+ feat`."""
    B = 2 * m
    per_set = 4 * B * C * h * w * 2
    nsets = max(2, int(np.ceil(target_mb * 1e6 / per_set)))
    g = torch.Generator().manual_seed(C + h + m)

    def cl():
        return torch.randn(B, C, h, w, generator=g).to(device, torch.float16).contiguous(memory_format=torch.channels_last)
    sets = [(cl(), cl(), cl(), cl()) for _ in range(nsets)]       # res, proj, feat, out

    def fused(i):
        res, proj, feat, out = sets[i % nsets]
        fused_ops.adapter_residual(res, proj, None, feat, out)

    def add(i):
        res, proj, _, out = sets[i % nsets]
        torch.add(proj, res, out=out)

    def add_feat(i):
        res, proj, feat, out = sets[i % nsets]
        torch.add(proj, res, out=out)
        out.add_(feat)

    out = {}
    for name, fn in (("fused_us", fused), ("torch_add_us", add), ("torch_add_then_feat_us", add_feat)):
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
    out["fused_bytes"] = 4 * B * C * h * w * 2                    # read a, b, feat; write out
    out["fused_share_of_hbm_bound"] = out["fused_bytes"] / HBM_BYTES_PER_S / (out["fused_us"] * 1e-6)
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--no-loop", action="store_true")
    ap.add_argument("--no-kernel", action="store_true")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_t2i_adapter.py needs a CUDA device (H100)")
    device = torch.device("cuda", 0)
    torch.cuda.set_device(device)
    torch.backends.cudnn.benchmark = True
    line = {"metric": "t2i_adapter_steps_per_sec_512sq_cfg", "unit": "steps/s, ms, us",
            "config": {"workload": bench.CONFIGS[2]["what"], "steps": STEPS, "cuda_graph": True, "rounds": args.rounds,
                       "adapters": "SD1.5-shaped full (cin 192, nums_rb 2) and light (nums_rb 4), seeded random "
                                   "weights, fp16; ControlNet SD1.5-shaped",
                       "kernel": "pww_adapter_residual_f16 at the SD1.5 512x512 level shapes, rows = 2m, feature on "
                                 "every row"},
            "device": bench.device_info(0)}
    with torch.no_grad():
        if not args.no_loop:
            line["loop"] = loop(device, args.rounds)
        if not args.no_kernel:
            ucfg = bench.unet_config(bench.CONFIGS[2]["unet"])
            sizes = unet_level_sizes(bench.CONFIGS[2]["size"] // 8, bench.CONFIGS[2]["size"] // 8)
            line["kernel"] = {f"m{m}": {f"C{c}_{h}x{w}": level_us(device, c, h, w, m)
                                        for c, (h, w) in zip(ucfg.block_out_channels, sizes)} for m in (1, 8)}
    print(json.dumps(line), flush=True)


if __name__ == "__main__":
    main()
