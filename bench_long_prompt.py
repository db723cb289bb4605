#!/usr/bin/env python
"""bench_long_prompt.py -- the workload of bench.py (default config: aurora_1 map, SD1.5-shaped UNet, 512x512, 30-step
LMS, CFG 7.5, fp16, one GPU) with a prompt that fills 1, 2 or 3 CLIP chunks, and the cross-attention kernels at the long
key counts.

    python bench_long_prompt.py [--prompt-chunks 2] [--steps 27] [--warmup 3] [--no-kernels]

One JSON line on stdout:
  value        denoising steps/s of one image (cond + uncond as one batch-2 UNet forward, CFG, LMS), inputs resident,
               CUDA-graph replay, CUDA-event time -- bench.py's `value`, with the longer prompt
  config       prompt_chunks and T (the text length the UNet's cross-attention sees)
  long_prompt  per T in {154, 231} at the N = 4096 level (8 heads of 40, cond + uncond, the aurora_1 map packed):
               one pww_xattn_fused_f16 launch, the dense pair (pww_xattn_stats_f16 + pww_xattn_fwd_f16) and the
               reference's inj_forward op sequence as eager torch fp16 (bench.eager_torch_xattn_us), in microseconds;
               alg_bytes = SURVEY 8d with the real T (Q, O, K, V in fp16 + 64 B of packed map per pixel + its index)
  device       name and power limit of the GPU the numbers were measured on
Writes nothing.
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

import bench  # noqa: E402  (workload definition, eager comparison, device info)
from paint_with_words_sd_b200.conditioning import _encode_text_color_inputs, pack_weight_map  # noqa: E402
from paint_with_words_sd_b200.scheduler import LMSDiscreteScheduler  # noqa: E402
from paint_with_words_sd_b200.synthetic import RandomTextEncoder, SimpleWordTokenizer  # noqa: E402
from paint_with_words_sd_b200.unet import build_unet  # noqa: E402
from tests.fixtures import SETTINGS, color_map_image  # noqa: E402

FILLER = ("intricate details, soft light, muted colours, fine brush strokes, calm atmosphere, wide shot, sharp focus, "
          "gentle shadows").split(" ")


def long_prompt(prompt: str, chunks: int, tok) -> str:
    """`prompt` extended with neutral style words until it needs `chunks` 77-token CLIP windows (75 prompt tokens each)."""
    if chunks == 1:
        return prompt
    words, i = prompt.split(" "), 0
    while len(tok(" ".join(words))["input_ids"]) - 2 <= 75 * (chunks - 1) + 40:
        words.append(FILLER[i % len(FILLER)])
        i += 1
    return " ".join(words)


def loop_steps_per_s(device, chunks: int, steps: int, warmup: int) -> dict:
    import paint_with_words_sd_b200 as P
    from paint_with_words_sd_b200.pipeline import PwWSampler, initial_latents
    cfg = bench.CONFIGS[2]
    size = cfg["size"]
    unet = build_unet(bench.unet_config(cfg["unet"]), seed=0, dtype=torch.float16, device=device)
    unet = unet.to(memory_format=torch.channels_last)
    P.patch_unet(unet)
    try:
        tok, enc = SimpleWordTokenizer(), RandomTextEncoder(cfg["text_dim"]).to(device)
        sch = LMSDiscreteScheduler(beta_start=0.00085, beta_end=0.012, beta_schedule="scaled_linear")
        sch.set_timesteps(cfg["sched_steps"])
        s = SETTINGS["aurora"]
        prompt = long_prompt(s["prompt"], chunks, tok)
        seeds, sep, cond, uncond = _encode_text_color_inputs(enc, tok, device, color_map_image("aurora", size),
                                                             dict(s["ctx"]), prompt, "", max_prompt_chunks=chunks)
        lat0 = (initial_latents((1, 4, size // 8, size // 8), 0, seeds, sep) * sch.init_noise_sigma).to(device)
        sampler = PwWSampler(unet, sch, [cond], [uncond], lat0, bench.weight_function, bench.GUIDANCE)

        def run(n):
            for _ in range(n):
                if sampler._step_no >= cfg["sched_steps"]:
                    sampler.restart(lat0)
                sampler.step()

        with torch.no_grad():
            run(warmup)
            torch.cuda.synchronize(device)
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            run(steps)
            e1.record()
            torch.cuda.synchronize(device)
        ms = e0.elapsed_time(e1)
        return {"value": steps / (ms / 1e3), "ms_per_step": ms / steps, "T": int(cond["CONTEXT_TENSOR"].shape[1]),
                "prompt_tokens": len(tok(prompt)["input_ids"]) - 2}
    finally:
        P.unpatch_all()


def long_map(T: int) -> torch.Tensor:
    """[4096, T] aurora_1 map of the 2-chunk long prompt (tests/golden/long_prompt.npz); at T = 231 its first chunk is
    repeated as the third (the same regions: the packed dictionary stays within 10 columns)."""
    w = torch.from_numpy(np.load(os.path.join(ROOT, "tests", "golden", "long_prompt.npz"))["w8"])
    return w if T == 154 else torch.cat([w, w[:, :77]], 1).contiguous()


def xattn_long(device, T: int, B=2, biased=1, H=8, D=40, target_mb=192, iters=64, reps=5) -> dict:
    """One pww_xattn_fused_f16 launch and the dense pair at T keys: CUDA events around a CUDA graph of back-to-back
    launches that cycle through buffer sets larger than L2 (bench.xattn_roofline's method)."""
    from paint_with_words_sd_b200 import _native
    L = _native.lib()
    N, C = 4096, H * D
    per_set = B * N * C * 2 * 2 + biased * N * 64
    nsets = max(2, int(math.ceil(target_mb * 1e6 / per_set)))
    g = torch.Generator(device="cpu").manual_seed(0)
    qs = [(torch.randn(B, N, C, generator=g) * 0.5).half().to(device) for _ in range(nsets)]
    outs = [torch.empty(B, N, C, dtype=torch.float16, device=device) for _ in range(nsets)]
    k = (torch.randn(B, T, C, generator=g) * 0.5).half().to(device)
    v = (torch.randn(B, T, C, generator=g) * 0.5).half().to(device)
    dense = torch.stack([long_map(T)] * biased, 0).contiguous()
    mp0, ci0 = pack_weight_map(dense)
    mps = [mp0.to(device).clone() for _ in range(nsets)]
    ci = ci0.to(device)
    ws = [dense.to(device).clone() for _ in range(min(nsets, 8))]
    idx = torch.tensor(list(range(biased)) + [-1] * (B - biased), dtype=torch.int32, device=device)
    stats = torch.zeros(B, dtype=torch.float32, device=device)
    gs = torch.full((1,), 0.4 * math.log(1 + 7.0), dtype=torch.float32, device=device)
    fws = torch.zeros(L.pww_xattn_fused_workspace_bytes(), dtype=torch.uint8, device=device)
    ws_bytes = L.pww_xattn_workspace_bytes(B, H, N, T, D)
    work = torch.zeros(ws_bytes, dtype=torch.uint8, device=device)
    scale = D ** -0.5

    def fused(i, stream):
        q, o, mp = qs[i % nsets], outs[i % nsets], mps[i % nsets]
        _native.check(L.pww_xattn_fused_f16(q.data_ptr(), k.data_ptr(), v.data_ptr(), o.data_ptr(), B, H, N, T, D,
                                            q.stride(0), q.stride(1), k.stride(0), k.stride(1), o.stride(0), o.stride(1),
                                            mp.data_ptr(), mp.stride(0), mp.shape[0], ci.data_ptr(), idx.data_ptr(), 0,
                                            gs.data_ptr(), scale, stats.data_ptr(), fws.data_ptr(), fws.numel(), stream),
                      "fused")

    def dstats(i, stream):
        q = qs[i % nsets]
        _native.check(L.pww_xattn_stats_f16(q.data_ptr(), k.data_ptr(), B, H, N, T, D, q.stride(0), q.stride(1),
                                            k.stride(0), k.stride(1), 0, idx.data_ptr(), stats.data_ptr(),
                                            work.data_ptr(), ws_bytes, stream), "stats")

    def dfwd(i, stream):
        q, o, w = qs[i % nsets], outs[i % nsets], ws[i % len(ws)]
        _native.check(L.pww_xattn_fwd_f16(q.data_ptr(), k.data_ptr(), v.data_ptr(), o.data_ptr(), B, H, N, T, D,
                                          q.stride(0), q.stride(1), k.stride(0), k.stride(1), o.stride(0), o.stride(1),
                                          w.data_ptr(), w.stride(0), idx.data_ptr(), stats.data_ptr(), gs.data_ptr(),
                                          scale, stream), "fwd")

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
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            torch.cuda.synchronize(device)
            e0.record()
            graph.replay()
            e1.record()
            torch.cuda.synchronize(device)
            best.append(e0.elapsed_time(e1) * 1e3 / iters)
        return float(np.median(best))

    us = timed(fused)
    alg = B * (2 * N * C * 2 + 2 * T * C * 2) + biased * (N * 64 + ci0.shape[-1])
    return {"us_per_launch": us, "alg_bytes_per_launch": alg, "achieved_GBps": alg / (us * 1e-6) / 1e9,
            "dense_pair_us": {"stats": timed(dstats), "fwd": timed(dfwd)},
            "eager_torch_fp16_us_per_cond_uncond_pair": bench.eager_torch_xattn_us(device, T=T)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--prompt-chunks", type=int, default=2, choices=[1, 2, 3])
    ap.add_argument("--steps", type=int, default=27)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--no-kernels", action="store_true", help="loop only: skip the long_prompt kernel timings")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_long_prompt.py needs a CUDA device (H100)")
    device = torch.device("cuda", 0)
    torch.cuda.set_device(device)
    torch.backends.cudnn.benchmark = True
    loop = loop_steps_per_s(device, args.prompt_chunks, args.steps, max(3, args.warmup))
    line = {"metric": bench.METRIC, "value": loop["value"], "unit": bench.UNIT, "ms_per_step": loop["ms_per_step"],
            "steps": args.steps, "config": {"workload": bench.CONFIGS[2]["what"], "prompt_chunks": args.prompt_chunks,
                                            "T": loop["T"], "prompt_tokens": loop["prompt_tokens"], "cuda_graph": True},
            "device": bench.device_info(0)}
    if not args.no_kernels:
        line["long_prompt"] = {}
        for T in (154, 231):
            line["long_prompt"][f"T{T}"] = xattn_long(device, T)
        line["long_prompt"]["note"] = "N=4096 C=320 H=8, B=2 (cond+uncond), one biased image"
    print(json.dumps(line), flush=True)


if __name__ == "__main__":
    main()
