"""Panoramas on the GPU: `pww_window_input` and `pww_window_update` bitwise against torch ops in the stated order,
chunk invariance, a one-window canvas against PwWSampler, PanoramaSampler against `tests/panorama_loop.py` on the CPU,
graphs, launch counts and the public API."""
import ctypes
import functools
import math

import pytest
import torch
from PIL import Image

import paint_with_words_sd_b200 as P
from oracle import loop as oracle_loop
from paint_with_words_sd_b200 import _native
from paint_with_words_sd_b200 import panorama as PN
from paint_with_words_sd_b200.conditioning import _encode_text_color_inputs
from paint_with_words_sd_b200.pipeline import _BETA, _SCALE, PwWSampler, _dtype_code, ancestral_noise
from paint_with_words_sd_b200.scheduler import (DPMSolverMultistepScheduler, EulerAncestralDiscreteScheduler,
                                                EulerDiscreteScheduler, LMSDiscreteScheduler)
from paint_with_words_sd_b200.synthetic import RandomTextEncoder, SimpleWordTokenizer
from paint_with_words_sd_b200.unet import UNetConfig, attention_modules, build_unet
from tests import panorama_loop
from tests.fixtures import SETTINGS, color_map_image

pytestmark = pytest.mark.gpu
WF = lambda w, sigma, qk: 0.4 * w * math.log(1 + sigma) * qk.max()   # noqa: E731
KW = dict(beta_start=0.00085, beta_end=0.012, beta_schedule="scaled_linear")
SAMPLERS = {"lms": LMSDiscreteScheduler, "euler": EulerDiscreteScheduler, "euler_a": EulerAncestralDiscreteScheduler,
            "dpmpp_2m": DPMSolverMultistepScheduler,
            "dpmpp_2m_karras": functools.partial(DPMSolverMultistepScheduler, use_karras_sigmas=True)}
DTYPES = {"fp32": torch.float32, "fp16": torch.float16, "bf16": torch.bfloat16}


def _scheduler(name, steps, prediction_type="epsilon"):
    sch = SAMPLERS[name](**KW, prediction_type=prediction_type)
    sch.set_timesteps(steps)
    return sch


def _sampler(name, h, w, window, stride, circular, per_chunk, steps=4, prediction_type="epsilon", unet=None,
             use_graph=False):
    """A PanoramaSampler over a random canvas with placeholder contexts: its step rows, noise and starts drive the
    kernels directly (it is never stepped unless `unet` is a real model)."""
    views = P.panorama_views(h, w, window, stride, circular)
    V = len(views[0]) * len(views[1])
    ctx = {"CONTEXT_TENSOR": torch.zeros(1, 77, 64)}
    sch = _scheduler(name, steps, prediction_type)
    lat = torch.randn(1, 4, h, w, generator=torch.manual_seed(h * 100 + w)) * float(sch.init_noise_sigma)
    return PN.PanoramaSampler(unet or torch.nn.Linear(1, 1), sch, [ctx] * V, [ctx] * V, lat.cuda(), views, window,
                              WF, 6.5, noise_seed=9, view_batch_size=per_chunk, use_graph=use_graph)


LAYOUTS = {   # (h, w, window, stride, circular): W % 4 == 0 or not, flush last windows, wrapped windows
    "flush48": (16, 48, 16, 4, False), "flush45": (16, 45, 16, 8, False),
    "circ48": (16, 48, 16, 8, True), "circ45_rows": (20, 45, 16, 7, True),
}


# ---- pww_window_input ----------------------------------------------------------------------------------------------
def _window_inputs(s, per_chunk_ins=None):
    """Run pww_window_input for every chunk of `s` at step 0: the list of [2k, 4, win, win] buffers."""
    L = _native.lib()
    s._params.copy_(s._rows[0])
    rows, cols = s._starts
    h, w = s.latents.shape[-2:]
    outs = []
    for first, x in zip(s._firsts, s._unet_ins):
        x = torch.full_like(x, float("nan"))
        _native.check(L.pww_window_input(s.latents.data_ptr(), s._params[_SCALE:].data_ptr(), rows.data_ptr(),
                                         rows.numel(), cols.data_ptr(), cols.numel(), first, x.shape[0] // 2,
                                         s.window, x.data_ptr(), _dtype_code(x.dtype), h, w, None), "pww_window_input")
        outs.append(x)
    torch.cuda.synchronize()
    return outs


@pytest.mark.parametrize("dtype", list(DTYPES))
@pytest.mark.parametrize("layout", list(LAYOUTS) + ["window13"])
@pytest.mark.parametrize("per_chunk", [1, 3, 64])
def test_window_input_is_a_scaled_gather(dtype, layout, per_chunk):
    h, w, window, stride, circular = LAYOUTS.get(layout, (20, 45, 13, 5, True))
    unet = torch.nn.Linear(1, 1).to("cuda", DTYPES[dtype])
    s = _sampler("lms", h, w, window, stride, circular, per_chunk, unet=unet)
    got = _window_inputs(s)
    scale = s._rows[0, _SCALE]
    crops = [(s.latents[0, :, r0:r0 + window][..., cols] * scale).to(DTYPES[dtype])
             for r0, cols in panorama_loop.windows_of(s.views, window, w)]
    for first, x in zip(s._firsts, got):
        k = x.shape[0] // 2
        want = torch.stack(crops[first:first + k])
        assert torch.equal(x[:k], want) and torch.equal(x[k:], want), first


# ---- pww_window_update ---------------------------------------------------------------------------------------------
def _outputs(s, dtype, layout, steps, seed):
    """Per step, the window outputs [V, 2, 4, win, win] (cond, uncond) in fp32 and the chunk tensors the UNet would
    return in `dtype` and `layout`."""
    g = torch.Generator().manual_seed(seed)
    V = sum(x.shape[0] // 2 for x in s._unet_ins)
    win = s.window
    per_step = []
    for _ in range(steps):
        e = (torch.randn(V, 2, 4, win, win, generator=g) + torch.linspace(-2, 2, V).view(V, 1, 1, 1, 1)).to(dtype)
        e[:, 1] *= 0.6
        chunks = []
        for first, x in zip(s._firsts, s._unet_ins):
            k = x.shape[0] // 2
            c = torch.cat([e[first:first + k, 0], e[first:first + k, 1]], 0).cuda()
            chunks.append(c.contiguous(memory_format=torch.channels_last) if layout == "channels_last" else c)
        per_step.append((e.float().cuda(), chunks))
    return per_step


def _kernel_run(s, per_step):
    L = _native.lib()
    lat, hist = s.latents.clone(), torch.zeros_like(s._derivs)
    rows, cols = s._starts
    h, w = lat.shape[-2:]
    for i, (_, chunks) in enumerate(per_step):
        p = s._rows[i].clone()
        table = (ctypes.c_void_p * len(chunks))(*[c.data_ptr() for c in chunks])
        _native.check(L.pww_window_update(table, len(chunks), s.m, _dtype_code(chunks[0].dtype), *chunks[0].stride(),
                                          rows.data_ptr(), rows.numel(), cols.data_ptr(), cols.numel(), s.window,
                                          lat.data_ptr(), hist.data_ptr(), s._hist_len,
                                          None if s._noise is None else s._noise.data_ptr(), s._gscale.data_ptr(),
                                          p[_BETA:].data_ptr(), p[s._form:].data_ptr(), h, w, None),
                      "pww_window_update")
    torch.cuda.synchronize()
    return lat, hist


def _torch_run(s, per_step):
    """The same steps as torch fp32 ops in the kernel's order."""
    lat, ring = s.latents.clone(), torch.zeros_like(s._derivs)
    L, win = ring.shape[0], s.window
    wins = panorama_loop.windows_of(s.views, win, lat.shape[-1])
    for i, (e, _) in enumerate(per_step):
        r = [float(v) for v in s._rows[i].tolist()]
        alpha, a, b, gamma, slot, nrow = r[s._form:s._form + 6]
        beta = r[_BETA:_BETA + 4]
        total, count = torch.zeros_like(lat), torch.zeros_like(lat)
        for v, (r0, cols) in enumerate(wins):
            g = e[v, 1] + s._gscale * (e[v, 0] - e[v, 1])
            seen = count[0, :, r0:r0 + win, cols] > 0
            total[0, :, r0:r0 + win, cols] = torch.where(seen, total[0, :, r0:r0 + win, cols] + g, g)
            count[0, :, r0:r0 + win, cols] += 1
        eps = total / count
        q = b * eps if a == 0 else a * lat + b * eps
        ring[int(slot)].copy_(q)
        acc = beta[0] * q
        for j in range(1, L):
            acc = acc + beta[j] * ring[(int(slot) - j) % L]
        lat = lat + acc if alpha == 1 else alpha * lat + acc
        if gamma != 0 and s._noise is not None:
            lat = lat + gamma * s._noise[int(nrow)]
    return lat, ring


UPDATE_CASES = [("lms", "epsilon"), ("euler", "epsilon"), ("euler_a", "epsilon"), ("dpmpp_2m", "epsilon"),
                ("euler", "v_prediction"), ("dpmpp_2m_karras", "v_prediction")]


@pytest.mark.parametrize("case", UPDATE_CASES, ids=[f"{n}-{p}" for n, p in UPDATE_CASES])
@pytest.mark.parametrize("dtype", list(DTYPES))
@pytest.mark.parametrize("out_layout", ["contiguous", "channels_last"])
@pytest.mark.parametrize("layout", list(LAYOUTS))
def test_window_update_is_the_stated_torch_ops_at_any_chunking(case, dtype, out_layout, layout):
    name, pred = case
    h, w, window, stride, circular = LAYOUTS[layout]
    steps = 4
    runs = []
    for per_chunk in (64, 2, 3):
        s = _sampler(name, h, w, window, stride, circular, per_chunk, steps, pred)
        per_step = _outputs(s, DTYPES[dtype], out_layout, steps, seed=h + w)
        lat, hist = _kernel_run(s, per_step)
        assert torch.isfinite(lat).all()
        runs.append((lat, hist))
        if per_chunk == 64:
            want_lat, want_hist = _torch_run(s, per_step)
            assert len(s._firsts) == 1
            assert torch.equal(lat, want_lat) and torch.equal(hist, want_hist)
        else:
            assert len(s._firsts) > 1
    for lat, hist in runs[1:]:                  # the same window outputs in 1, and in 2 or more, chunks: the same bits
        assert torch.equal(lat, runs[0][0]) and torch.equal(hist, runs[0][1])


# ---- the sampler ---------------------------------------------------------------------------------------------------
def wide_color_map(names=("aurora", "cat_dog", "aurora"), size=128) -> Image.Image:
    out = Image.new("RGB", (len(names) * size, size))
    for i, n in enumerate(names):
        out.paste(color_map_image(n, size), (i * size, 0))
    return out


def _tiny(dtype=torch.float16, device="cuda"):
    return build_unet(UNetConfig.tiny(), seed=0, dtype=dtype, device=device)


@pytest.mark.parametrize("dtype", ["fp16", "bf16"])
@pytest.mark.parametrize("name", list(SAMPLERS))
def test_one_window_canvas_is_pwwsampler(name, dtype):
    s = SETTINGS["aurora"]
    unet = _tiny(DTYPES[dtype])
    _, _, cond, uncond = _encode_text_color_inputs(RandomTextEncoder(64).cuda(), SimpleWordTokenizer(), "cuda",
                                                   color_map_image("aurora", 128), dict(s["ctx"]), s["prompt"], "")
    lat = (torch.randn(1, 4, 16, 16, generator=torch.manual_seed(0)) * 14.6).cuda()
    try:
        P.patch_unet(unet)
        pano = PN.PanoramaSampler(unet, _scheduler(name, 5), [cond], [uncond], lat, ([0], [0]), 16, WF, 7.5,
                                  noise_seed=4).run()
        plain = PwWSampler(unet, _scheduler(name, 5), [cond], [uncond], lat, WF, 7.5, noise_seed=4).run()
    finally:
        P.unpatch_all()
    assert torch.isfinite(pano).all() and torch.equal(pano, plain)


PANO_CASES = [(n, stride, circ) for n in ("lms", "dpmpp_2m", "euler_a") for stride in (4, 8) for circ in (False, True)]


def _pano_inputs(device, stride, circular):
    s = SETTINGS["aurora"]
    views = P.panorama_views(16, 48, 16, stride, circular)
    conds, unconds = PN.panorama_conditioning(RandomTextEncoder(64).to(device), SimpleWordTokenizer(), device,
                                              wide_color_map(), dict(s["ctx"]), s["prompt"], "", views, 16)
    return views, conds, unconds


@pytest.mark.parametrize("case", PANO_CASES, ids=[f"{n}-s{st}-{'circ' if c else 'flat'}" for n, st, c in PANO_CASES])
def test_sampler_matches_the_multidiffusion_loop(case):
    name, stride, circular = case
    steps = 3
    lat = torch.randn(1, 4, 16, 48, generator=torch.manual_seed(2)) * 14.6
    views, conds, unconds = _pano_inputs("cpu", stride, circular)
    unet = build_unet(UNetConfig.tiny(), seed=0)
    try:
        oracle_loop.patch_with_oracle(unet)
        noise = ancestral_noise([6], (4, 16, 48), steps) if name == "euler_a" else None
        ref = panorama_loop.reference_panorama_loop(unet, _scheduler(name, steps), conds, unconds, lat, views, 16, WF,
                                                    7.5, noise=noise)
    finally:
        cls = attention_modules(unet)[0].__class__
        if "__call__" in cls.__dict__:
            delattr(cls, "__call__")
    views, conds, unconds = _pano_inputs("cuda", stride, circular)
    unet = _tiny()
    try:
        P.patch_unet(unet)
        out = PN.PanoramaSampler(unet, _scheduler(name, steps), conds, unconds, lat.cuda(), views, 16, WF, 7.5,
                                 noise_seed=6, view_batch_size=4).run().float().cpu()
    finally:
        P.unpatch_all()
    d = (out - ref).abs().max().item()
    assert torch.isfinite(out).all() and d <= 2e-2 * ref.abs().max().item(), d


def _tiny_run(view_batch_size, use_graph=True, name="lms"):
    views, conds, unconds = _pano_inputs("cuda", 4, True)
    unet = _tiny()
    lat = (torch.randn(1, 4, 16, 48, generator=torch.manual_seed(2)) * 14.6).cuda()
    try:
        P.patch_unet(unet)
        s = PN.PanoramaSampler(unet, _scheduler(name, 4), conds, unconds, lat, views, 16, WF, 7.5, noise_seed=1,
                               view_batch_size=view_batch_size, use_graph=use_graph)
        return s.run().clone(), s
    finally:
        P.unpatch_all()


def test_chunking_changes_only_fp16_noise_and_graphs_replay_eager_bits():
    one, s1 = _tiny_run(64)
    many, sk = _tiny_run(1)
    assert len(s1._firsts) == 1 and len(sk._firsts) == 12
    d = (one - many).abs().max().item()
    assert d <= 1e-2 * one.abs().max().item(), d
    for name in ("lms", "euler_a"):
        assert torch.equal(_tiny_run(5, True, name)[0], _tiny_run(5, False, name)[0])


class _TorchUNet(torch.nn.Module):
    """A UNet stand-in made of torch ops only, so a step's native launches are the sampler's own."""

    def __init__(self):
        super().__init__()
        self.conv = torch.nn.Conv2d(4, 4, 3, padding=1).cuda()

    def forward(self, x, t, encoder_hidden_states=None):
        class _Out:
            sample = torch.tanh(self.conv(x.float()))
        return _Out()


def test_launch_counts():
    for per_chunk, chunks in ((64, 1), (4, 3), (1, 12)):
        s = _sampler("dpmpp_2m", 16, 48, 16, 4, True, per_chunk, unet=_TorchUNet(), use_graph=True)
        s.run(1)
        assert s.native_launches_per_step == chunks + 1
    views, conds, unconds = _pano_inputs("cuda", 4, True)
    s = SETTINGS["aurora"]
    _, _, cond, uncond = _encode_text_color_inputs(RandomTextEncoder(64).cuda(), SimpleWordTokenizer(), "cuda",
                                                   color_map_image("aurora", 128), dict(s["ctx"]), s["prompt"], "")
    unet = _tiny()
    try:
        P.patch_unet(unet)
        lat = torch.randn(1, 4, 16, 16).cuda()
        plain = PwWSampler(unet, _scheduler("lms", 2), [cond], [uncond], lat, WF)
        plain.run(1)
        one = PN.PanoramaSampler(unet, _scheduler("lms", 2), [cond], [uncond], lat, ([0], [0]), 16, WF)
        one.run(1)
        assert one.native_launches_per_step == plain.native_launches_per_step
        unet_launches = plain.native_launches_per_step - 2
        for per_chunk, k in ((4, 3), (5, 3), (12, 1)):
            pano = PN.PanoramaSampler(unet, _scheduler("lms", 2), conds, unconds, torch.randn(1, 4, 16, 48).cuda(),
                                      views, 16, WF, view_batch_size=per_chunk)
            pano.run(1)
            assert pano.native_launches_per_step == k * (1 + unet_launches) + 1, per_chunk
    finally:
        P.unpatch_all()


# ---- the public API ------------------------------------------------------------------------------------------------
def test_public_panorama_sd15_fp16():
    a = SETTINGS["aurora"]
    cm = wide_color_map(("aurora", "cat_dog"), 512)
    ctx = dict(a["ctx"])
    ctx[(7, 9, 182)] = "aurora,0.5,11"                  # regional seeding
    tools = P.pww_load_tools("cuda:0", hf_model_path="synthetic:sd15")
    try:
        run = functools.partial(P.paint_with_words_panorama, ctx, cm, a["prompt"], num_inference_steps=3,
                                weight_function=WF, preloaded_utils=tools, seed=3)
        image = run()
        first, second = run(return_latents=True), run(return_latents=True)
    finally:
        P.unpatch_all()
    assert image.size == cm.size == (1024, 512)
    assert tuple(first.shape) == (1, 4, 64, 128) and torch.isfinite(first).all() and torch.equal(first, second)


def test_public_panorama_tiny_bf16_vpred_circular():
    a = SETTINGS["cat_dog"]
    cm = wide_color_map()
    tools = P.pww_load_tools("cuda:0", hf_model_path="synthetic:tiny", torch_dtype=torch.bfloat16,
                             prediction_type="v_prediction", scheduler_type=EulerAncestralDiscreteScheduler)
    assert tools[4].config["prediction_type"] == "v_prediction"
    try:
        run = functools.partial(P.paint_with_words_panorama, dict(a["ctx"]), cm, a["prompt"], num_inference_steps=4,
                                weight_function=WF, preloaded_utils=tools, seed=8, circular_padding=True,
                                view_batch_size=2, max_prompt_chunks=2)
        image = run()
        first, second = run(return_latents=True), run(return_latents=True)
    finally:
        P.unpatch_all()
    assert image.size == cm.size == (384, 128)
    assert tuple(first.shape) == (1, 4, 16, 48) and torch.isfinite(first).all() and torch.equal(first, second)
