#!/usr/bin/env python
"""bench_batch.py -- differently configured images in one sampler against one sampler per image, and the per-image
(`_multi`) one-launch kernel against one launch per image.

    python bench_batch.py [--ks 1,2,4,8] [--reps 3] [--no-loop] [--no-kernels]

Loop: bench.py's default workload (aurora_1 map, SD1.5-shaped UNet, 512x512, 30-step LMS, fp16, CUDA graph).  Image i
has seed i, the weight function WEIGHT_FUNCTIONS[i % 3] (the README's comparison grid: 0.4*w*log(1+sigma)*max,
0.4*w*log(1+sigma)*std, 0.4*w*log(1+sigma^2)*std) and the guidance scale GUIDANCE_SCALES[i % 2].  For each k, k images
run as ONE PwWSampler (a 2k UNet batch) and as k single-image samplers one after another; both are timed over the whole
30-step schedule after a warm-up pass (graph capture) with CUDA events, median of --reps runs.

Kernels: N = 4096, 8 heads of 40 (the 64x64 level), T = 77 and 231, aurora_1 maps packed.  One pww_xattn_fused_multi_f16
launch over k cond + k uncond images with mixed kinds and G against k pww_xattn_fused_f16 launches of one cond + uncond
pair each, and the uniform `_multi` launch against pww_xattn_fused_f16 at B = 2.  CUDA events around a CUDA graph of
back-to-back launches that cycle through buffer sets larger than L2 (bench.xattn_roofline's method).

One JSON line on stdout, with the GPU's name and power limit.  Writes nothing.
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

import bench  # noqa: E402  (workload definition, golden maps, device info)
import bench_long_prompt  # noqa: E402  (the T = 231 map)
from paint_with_words_sd_b200.conditioning import _encode_text_color_inputs, pack_weight_map  # noqa: E402
from paint_with_words_sd_b200.scheduler import LMSDiscreteScheduler  # noqa: E402
from paint_with_words_sd_b200.synthetic import RandomTextEncoder, SimpleWordTokenizer  # noqa: E402
from paint_with_words_sd_b200.unet import build_unet  # noqa: E402
from tests.fixtures import SETTINGS, color_map_image  # noqa: E402


def wf_max(w, sigma, qk):
    return 0.4 * w * math.log(1 + sigma) * qk.max()


def wf_std(w, sigma, qk):
    return 0.4 * w * math.log(1 + sigma) * qk.std()


def wf_std_sq(w, sigma, qk):
    return 0.4 * w * math.log(1 + sigma ** 2) * qk.std()


WEIGHT_FUNCTIONS = (wf_max, wf_std, wf_std_sq)
GUIDANCE_SCALES = (7.5, 5.0)


def _events_ms(fn) -> float:
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    e0.record()
    fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1)


def loop_images_per_s(device, ks, reps: int) -> dict:
    import paint_with_words_sd_b200 as P
    from paint_with_words_sd_b200.pipeline import PwWSampler, initial_latents
    cfg = bench.CONFIGS[2]
    size, steps = cfg["size"], cfg["sched_steps"]
    unet = build_unet(bench.unet_config(cfg["unet"]), seed=0, dtype=torch.float16, device=device)
    unet = unet.to(memory_format=torch.channels_last)
    P.patch_unet(unet)
    try:
        tok, enc = SimpleWordTokenizer(), RandomTextEncoder(cfg["text_dim"]).to(device)
        sch = LMSDiscreteScheduler(beta_start=0.00085, beta_end=0.012, beta_schedule="scaled_linear")
        sch.set_timesteps(steps)
        s = SETTINGS["aurora"]
        images = []
        for i in range(max(ks)):
            seeds, sep, cond, uncond = _encode_text_color_inputs(enc, tok, device, color_map_image("aurora", size),
                                                                 dict(s["ctx"]), s["prompt"], "")
            lat = (initial_latents((1, 4, size // 8, size // 8), i, seeds, sep) * sch.init_noise_sigma).to(device)
            images.append((cond, uncond, lat, WEIGHT_FUNCTIONS[i % 3], GUIDANCE_SCALES[i % 2]))

        def full_run(sampler, lat0):
            sampler.restart(lat0)
            for _ in range(steps):
                sampler.step()

        res = {}
        with torch.no_grad():
            for k in ks:
                part = images[:k]
                lat = torch.cat([x[2] for x in part], 0)
                batched = PwWSampler(unet, sch, [x[0] for x in part], [x[1] for x in part], lat,
                                     [x[3] for x in part], [x[4] for x in part])
                solo = [PwWSampler(unet, sch, [x[0]], [x[1]], x[2], x[3], x[4]) for x in part]
                full_run(batched, lat)                              # warm-up: graph capture, library autotune
                for smp, x in zip(solo, part):
                    full_run(smp, x[2])
                t_b, t_s = [], []
                for _ in range(reps):                               # alternate the two arms
                    t_b.append(_events_ms(lambda: full_run(batched, lat)))
                    t_s.append(_events_ms(lambda: [full_run(smp, x[2]) for smp, x in zip(solo, part)]))
                mb, ms = float(np.median(t_b)), float(np.median(t_s))
                res[f"k{k}"] = {"batched_images_per_s": k / (mb / 1e3), "sequential_images_per_s": k / (ms / 1e3),
                                "batched_ms": mb, "sequential_ms": ms, "speedup": ms / mb,
                                "native_launches_per_step": {"batched": batched.native_launches_per_step,
                                                             "solo": solo[0].native_launches_per_step}}
                del batched, solo
                torch.cuda.empty_cache()
        return res
    finally:
        P.unpatch_all()


def _map(T: int) -> torch.Tensor:
    return bench.golden_weight_map(4096) if T == 77 else bench_long_prompt.long_map(T)


def xattn_multi(device, k: int, T: int, H=8, D=40, target_mb=192, iters=64, reps=5) -> dict:
    """Per group of k cond + uncond pairs: one mixed `_multi` launch vs k pww_xattn_fused_f16 launches at B = 2.  The
    batch is laid out in pairs [c0, u0, c1, u1, ...], so pair j is a contiguous B = 2 slice for the per-pair launch."""
    from paint_with_words_sd_b200 import _native
    L = _native.lib()
    N, C, B = 4096, H * D, 2 * k
    per_set = B * N * C * 2 * 2 + k * N * 64
    nsets = max(2, int(math.ceil(target_mb * 1e6 / per_set)))
    g = torch.Generator(device="cpu").manual_seed(0)
    qs = [(torch.randn(B, N, C, generator=g) * 0.5).half().to(device) for _ in range(nsets)]
    outs = [torch.empty(B, N, C, dtype=torch.float16, device=device) for _ in range(nsets)]
    kk = (torch.randn(B, T, C, generator=g) * 0.5).half().to(device)
    vv = (torch.randn(B, T, C, generator=g) * 0.5).half().to(device)
    mp0, ci0 = pack_weight_map(torch.stack([_map(T)] * k, 0).contiguous())
    mps = [mp0.to(device).clone() for _ in range(nsets)]
    ci = ci0.to(device)
    idx = torch.tensor([j // 2 if j % 2 == 0 else -1 for j in range(B)], dtype=torch.int32, device=device)
    idx1 = torch.tensor([0, -1], dtype=torch.int32, device=device)
    kinds = torch.tensor([(j // 2) % 2 if j % 2 == 0 else 0 for j in range(B)], dtype=torch.int32, device=device)
    gvals = torch.tensor([0.4 * math.log(1 + 7.0 ** (1 + (j // 2) % 2)) for j in range(B)], dtype=torch.float32,
                         device=device)
    uni_kinds = torch.zeros(2, dtype=torch.int32, device=device)
    uni_g = torch.full((2,), 0.4 * math.log(1 + 7.0), dtype=torch.float32, device=device)
    stats = torch.zeros(B, dtype=torch.float32, device=device)
    fws = torch.zeros(L.pww_xattn_fused_workspace_bytes(), dtype=torch.uint8, device=device)
    scale = D ** -0.5

    def call(fn, q, o, mp, b0, nb, ix, stat, gp, stream):
        off_q, off_k = b0 * q.stride(0) * 2, b0 * kk.stride(0) * 2
        _native.check(fn(q.data_ptr() + off_q, kk.data_ptr() + off_k, vv.data_ptr() + off_k, o.data_ptr() + off_q, nb,
                         H, N, T, D, q.stride(0), q.stride(1), kk.stride(0), kk.stride(1), o.stride(0), o.stride(1),
                         mp.data_ptr() + (b0 // 2) * mp.stride(0) * 2, mp.stride(0), mp.shape[0] - b0 // 2,
                         ci.data_ptr() + (b0 // 2) * ci.stride(0), ix, stat, gp, scale, stats.data_ptr() + b0 * 4,
                         fws.data_ptr(), fws.numel(), stream), fn.__name__)

    def multi(i, stream):
        call(L.pww_xattn_fused_multi_f16, qs[i % nsets], outs[i % nsets], mps[i % nsets], 0, B, idx.data_ptr(),
             kinds.data_ptr(), gvals.data_ptr(), stream)

    def per_pair(i, stream):
        for j in range(k):
            call(L.pww_xattn_fused_f16, qs[i % nsets], outs[i % nsets], mps[i % nsets], 2 * j, 2, idx1.data_ptr(),
                 j % 2, gvals.data_ptr() + 2 * j * 4, stream)

    def uniform_multi(i, stream):
        call(L.pww_xattn_fused_multi_f16, qs[i % nsets], outs[i % nsets], mps[i % nsets], 0, 2, idx1.data_ptr(),
             uni_kinds.data_ptr(), uni_g.data_ptr(), stream)

    def single(i, stream):
        call(L.pww_xattn_fused_f16, qs[i % nsets], outs[i % nsets], mps[i % nsets], 0, 2, idx1.data_ptr(), 0,
             uni_g.data_ptr(), stream)

    def timed(fn):
        s = torch.cuda.Stream(device=device)
        with torch.cuda.stream(s):
            for i in range(3):
                fn(i, s.cuda_stream)
        s.synchronize()
        graph = torch.cuda.CUDAGraph()
        with torch.cuda.graph(graph, stream=s):
            for i in range(iters):
                fn(i, torch.cuda.current_stream(device).cuda_stream)
        best = []
        for _ in range(reps):
            best.append(_events_ms(graph.replay) * 1e3 / iters)
        return float(np.median(best))

    t_multi, t_pairs = timed(multi), timed(per_pair)
    res = {"multi_us": t_multi, "per_pair_launches_us": t_pairs, "multi_us_per_image": t_multi / k,
           "per_pair_us_per_image": t_pairs / k}
    if k == 1:
        res["uniform_multi_B2_us"], res["fused_f16_B2_us"] = timed(uniform_multi), timed(single)
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--ks", default="1,2,4,8", help="images per sampler / cond+uncond pairs per launch")
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--no-loop", action="store_true")
    ap.add_argument("--no-kernels", action="store_true")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_batch.py needs a CUDA device (H100)")
    ks = [int(x) for x in args.ks.split(",")]
    device = torch.device("cuda", 0)
    torch.cuda.set_device(device)
    torch.backends.cudnn.benchmark = True
    line = {"metric": "images_per_sec_512sq_cfg_30steps", "unit": "images/s",
            "config": {"workload": bench.CONFIGS[2]["what"],
                       "weight_functions": ["0.4*w*log(1+sigma)*max", "0.4*w*log(1+sigma)*std",
                                            "0.4*w*log(1+sigma^2)*std"],
                       "guidance_scales": list(GUIDANCE_SCALES), "cuda_graph": True, "reps": args.reps},
            "device": bench.device_info(0)}
    if not args.no_loop:
        line["loop"] = loop_images_per_s(device, ks, args.reps)
    if not args.no_kernels:
        line["kernels"] = {f"T{T}": {f"k{k}": xattn_multi(device, k, T) for k in ks} for T in (77, 231)}
        line["kernels"]["note"] = ("N=4096 C=320 H=8; per group of k cond+uncond pairs: one mixed _multi launch vs k "
                                   "pww_xattn_fused_f16 launches; at k=1 also uniform _multi vs pww_xattn_fused_f16")
    print(json.dumps(line), flush=True)


if __name__ == "__main__":
    main()
