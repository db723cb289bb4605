#!/usr/bin/env python
"""bench_dtype.py -- fp16 against bf16 UNets on the default workload, and the one-launch cross-attention in both types.

    python bench_dtype.py [--rounds 3] [--no-loop] [--no-kernel]

Loop: bench.py's default workload (aurora_1 map, SD1.5-shaped UNet, 512x512, 30 LMS steps, CFG 7.5, CUDA graph, one
image per sampler) with an fp16 and a bf16 UNet built from the same seeded weights.  Each run is timed whole after a
warm-up pass (graph capture) with CUDA events; the two types alternate for --rounds rounds and each gets the median
steps/s, its range and the SM clock nvidia-smi sampled during each window.  The relative RMSE between the two types'
final latents is reported for information only: bf16 keeps 8 significand bits against fp16's 11, so it is expected to be
larger than the fp16 run's distance to an fp32 one.

Kernel: one pww_xattn_fused_{f16,bf16} launch at N = 4096, 8 heads of 40, 77 keys, cond + uncond halves (B = 2 and
B = 16), microseconds per launch from CUDA events around a CUDA graph of back-to-back launches that cycle through more
than L2 of buffers, as bench.py's roofline leg does.

One JSON line on stdout, with the GPU's name, power limit and SM clock.  Writes nothing.
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

import bench  # noqa: E402  (workload definition, device info, clock sampler, weight maps)
from paint_with_words_sd_b200 import _native  # noqa: E402
from paint_with_words_sd_b200.conditioning import _encode_text_color_inputs, pack_weight_map  # noqa: E402
from paint_with_words_sd_b200.scheduler import LMSDiscreteScheduler  # noqa: E402
from paint_with_words_sd_b200.synthetic import RandomTextEncoder, SimpleWordTokenizer  # noqa: E402
from paint_with_words_sd_b200.unet import build_unet  # noqa: E402
from tests.fixtures import SETTINGS, color_map_image  # noqa: E402

DTYPES = {"fp16": torch.float16, "bf16": torch.bfloat16}
STEPS = 30


def _events_ms(fn) -> float:
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    e0.record()
    fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1)


def loop(device, rounds: int) -> dict:
    import paint_with_words_sd_b200 as P
    from paint_with_words_sd_b200.pipeline import PwWSampler, initial_latents
    cfg = bench.CONFIGS[2]
    size = cfg["size"]
    tok, enc = SimpleWordTokenizer(), RandomTextEncoder(cfg["text_dim"]).to(device)
    s = SETTINGS["aurora"]
    seeds, sep, cond, uncond = _encode_text_color_inputs(enc, tok, device, color_map_image("aurora", size),
                                                         dict(s["ctx"]), s["prompt"], "")
    lat0 = initial_latents((1, 4, size // 8, size // 8), 0, seeds, sep)
    runs, final = {}, {}
    try:
        for name, dt in DTYPES.items():
            unet = build_unet(bench.unet_config(cfg["unet"]), seed=0, dtype=dt, device=device)
            unet = unet.to(memory_format=torch.channels_last)
            P.patch_unet(unet)
            sch = LMSDiscreteScheduler(beta_start=0.00085, beta_end=0.012, beta_schedule="scaled_linear")
            sch.set_timesteps(STEPS)
            lat = (lat0 * sch.init_noise_sigma).to(device)
            smp = PwWSampler(unet, sch, [cond], [uncond], lat, bench.weight_function, bench.GUIDANCE)

            def run(smp=smp, lat=lat):
                smp.restart(lat)
                for _ in range(STEPS):
                    smp.step()
            run()                                               # warm-up: graph capture, library autotune
            final[name] = smp.latents.float().clone()
            runs[name] = (smp, run)
        times = {n: [] for n in DTYPES}
        clocks = {n: [] for n in DTYPES}
        for _ in range(rounds):                                 # alternating: drift of the card hits both types
            for name in DTYPES:
                with bench.ClockSampler(device.index or 0) as clk:
                    times[name].append(_events_ms(runs[name][1]))
                clocks[name].append(clk.summary())
    finally:
        P.unpatch_all()
    res = {}
    for name in DTYPES:
        t = times[name]
        res[name] = {"steps_per_s": STEPS / (float(np.median(t)) / 1e3),
                     "steps_per_s_range": [STEPS / (max(t) / 1e3), STEPS / (min(t) / 1e3)],
                     "native_launches_per_step": runs[name][0].native_launches_per_step,
                     "sm_mhz": [c["sm_mhz"] for c in clocks[name]],
                     "clock_reasons": sorted({r for c in clocks[name] for r in c["reasons"]})}
    a, b = final["bf16"], final["fp16"]
    res["rel_rmse_bf16_vs_fp16_latents"] = ((a - b).pow(2).mean().sqrt() / b.pow(2).mean().sqrt()).item()
    return res


def fused_launch_us(device, dtype, B: int, biased: int, N=4096, H=8, D=40, T=77, target_mb=192, iters=64,
                    reps=5) -> float:
    """Microseconds per pww_xattn_fused launch of `dtype` over back-to-back launches cycling through > L2 of buffers."""
    L = _native.lib()
    fn = getattr(L, "pww_xattn_fused_bf16" if dtype == torch.bfloat16 else "pww_xattn_fused_f16")
    C = H * D
    nsets = max(2, int(math.ceil(target_mb * 1e6 / (B * N * C * 2 * 2 + biased * N * 64))))
    g = torch.Generator().manual_seed(0)
    qs = [(torch.randn(B, N, C, generator=g) * 0.5).to(device, dtype) for _ in range(nsets)]
    outs = [torch.empty(B, N, C, dtype=dtype, device=device) for _ in range(nsets)]
    k = (torch.randn(B, T, C, generator=g) * 0.5).to(device, dtype)
    v = (torch.randn(B, T, C, generator=g) * 0.5).to(device, dtype)
    base = bench.golden_weight_map(N)
    mp0, ci0 = pack_weight_map(torch.stack([base] * biased, 0).contiguous())
    mps = [mp0.to(device).clone() for _ in range(nsets)]
    ci = ci0.to(device)
    idx = torch.tensor(list(range(biased)) + [-1] * (B - biased), dtype=torch.int32, device=device)
    stats = torch.zeros(B, dtype=torch.float32, device=device)
    gs = torch.full((1,), 0.4 * math.log(1 + 7.0), dtype=torch.float32, device=device)
    ws = torch.zeros(L.pww_xattn_fused_workspace_bytes(), dtype=torch.uint8, device=device)

    def launch(i):
        q, o, mp = qs[i % nsets], outs[i % nsets], mps[i % nsets]
        rc = fn(q.data_ptr(), k.data_ptr(), v.data_ptr(), o.data_ptr(), B, H, N, T, D, q.stride(0), q.stride(1),
                k.stride(0), k.stride(1), o.stride(0), o.stride(1), mp.data_ptr(), mp.stride(0), mp.shape[0],
                ci.data_ptr(), idx.data_ptr(), _native.PWW_STAT_MAX, gs.data_ptr(), D ** -0.5, stats.data_ptr(),
                ws.data_ptr(), ws.numel(), torch.cuda.current_stream(device).cuda_stream)
        _native.check(rc, fn.__name__)

    s = torch.cuda.Stream(device=device)
    with torch.cuda.stream(s):
        for i in range(3):
            launch(i)
    s.synchronize()
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph, stream=s):
        for i in range(iters):
            launch(i)
    return float(np.median([_events_ms(graph.replay) * 1e3 / iters for _ in range(reps)]))


def kernel(device, rounds: int) -> dict:
    res = {}
    for B, biased in ((2, 1), (16, 8)):
        t = {n: [] for n in DTYPES}
        for _ in range(rounds):
            for name, dt in DTYPES.items():
                t[name].append(fused_launch_us(device, dt, B, biased))
        res[f"B{B}"] = {f"{n}_us": float(np.median(v)) for n, v in t.items()}
        res[f"B{B}"].update({f"{n}_us_range": [min(v), max(v)] for n, v in t.items()})
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--no-loop", action="store_true")
    ap.add_argument("--no-kernel", action="store_true")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_dtype.py needs a CUDA device (H100)")
    device = torch.device("cuda", 0)
    torch.cuda.set_device(device)
    torch.backends.cudnn.benchmark = True
    line = {"metric": "fp16_vs_bf16_steps_per_sec_512sq_cfg", "unit": "steps/s, us",
            "config": {"workload": bench.CONFIGS[2]["what"], "steps": STEPS, "cuda_graph": True, "rounds": args.rounds,
                       "kernel": "pww_xattn_fused N=4096 H=8 D=40 T=77, B=2 (1 biased) and B=16 (8 biased)"},
            "device": bench.device_info(0)}
    with torch.no_grad():
        if not args.no_loop:
            line["loop"] = loop(device, args.rounds)
        if not args.no_kernel:
            line["kernel"] = kernel(device, args.rounds)
    print(json.dumps(line), flush=True)


if __name__ == "__main__":
    main()
