"""Panoramas on the CPU: the window layout, per-window conditioning, the canvas start latents, the C entry points'
argument checks, and the self-checks of `tests/panorama_loop.py` (diffusers' MultiDiffusion loop restated)."""
import ctypes
import functools
import math

import numpy as np
import pytest
import torch
from PIL import Image

import paint_with_words_sd_b200 as P
from oracle import loop as oracle_loop
from paint_with_words_sd_b200 import _native
from paint_with_words_sd_b200 import panorama as PN
from paint_with_words_sd_b200.conditioning import _encode_text_color_inputs
from paint_with_words_sd_b200.pipeline import ancestral_noise, initial_latents
from paint_with_words_sd_b200.scheduler import (DPMSolverMultistepScheduler, EulerAncestralDiscreteScheduler,
                                                EulerDiscreteScheduler, LMSDiscreteScheduler)
from paint_with_words_sd_b200.synthetic import RandomTextEncoder, SimpleWordTokenizer
from paint_with_words_sd_b200.unet import UNetConfig, attention_modules, build_unet
from tests import panorama_loop
from tests.fixtures import SETTINGS, color_map_image

WF = lambda w, sigma, qk: 0.4 * w * math.log(1 + sigma) * qk.max()   # noqa: E731
KW = dict(beta_start=0.00085, beta_end=0.012, beta_schedule="scaled_linear")
SAMPLERS = {"lms": LMSDiscreteScheduler, "euler": EulerDiscreteScheduler, "euler_a": EulerAncestralDiscreteScheduler,
            "dpmpp_2m": DPMSolverMultistepScheduler,
            "dpmpp_2m_karras": functools.partial(DPMSolverMultistepScheduler, use_karras_sigmas=True)}


def wide_color_map(size: int = 128) -> Image.Image:
    """Two colour-map fixtures side by side: [size, 2 size] pixels."""
    out = Image.new("RGB", (2 * size, size))
    out.paste(color_map_image("aurora", size), (0, 0))
    out.paste(color_map_image("cat_dog", size), (size, 0))
    return out


# ---- window layout -------------------------------------------------------------------------------------------------
def test_views_of_a_512x2048_canvas_at_stride_8():
    rows, cols = P.panorama_views(64, 256, 64, 8)
    assert rows == [0] and cols == list(range(0, 193, 8)) and len(cols) == 25


def test_views_add_a_window_flush_with_the_edge():
    assert P.panorama_views(64, 100, 64, 16) == ([0], [0, 16, 32, 36])
    assert P.panorama_views(100, 64, 64, 16) == ([0, 16, 32, 36], [0])
    assert P.panorama_views(64, 64, 64, 8) == ([0], [0])            # one window
    assert P.panorama_views(16, 48, 16, 4)[1] == list(range(0, 33, 4))


def test_circular_views_wrap_the_columns_only():
    rows, cols = P.panorama_views(80, 100, 64, 16, circular=True)
    assert rows == [0, 16] and cols == [0, 16, 32, 48, 64, 80, 96]
    assert P.panorama_views(16, 48, 16, 8, circular=True) == ([0], [0, 8, 16, 24, 32, 40])


def _brute_force_count(h, w, window, rows, cols, circular):
    count = np.zeros((h, w), int)
    for y in range(h):
        for x in range(w):
            for r0 in rows:
                for c0 in cols:
                    dx = (x - c0) % w if circular else x - c0
                    count[y, x] += (0 <= y - r0 < window) and (0 <= dx < window)
    return count


@pytest.mark.parametrize("h,w,window,stride,circular", [(16, 48, 16, 4, False), (16, 48, 16, 8, True),
                                                         (20, 37, 16, 5, False), (20, 37, 16, 7, True),
                                                         (24, 24, 8, 8, False), (13, 50, 13, 13, True)])
def test_every_canvas_value_is_covered(h, w, window, stride, circular):
    rows, cols = P.panorama_views(h, w, window, stride, circular)
    count = np.zeros((h, w), int)
    for r0, c in panorama_loop.windows_of((rows, cols), window, w):
        count[r0:r0 + window, c.numpy()] += 1
    assert (count >= 1).all()
    np.testing.assert_array_equal(count, _brute_force_count(h, w, window, rows, cols, circular))


@pytest.mark.parametrize("args,match", [((64, 256, 64, 0), "stride"), ((64, 256, 64, 65), "stride"),
                                        ((32, 256, 64, 8), "smaller"), ((64, 40, 64, 8), "smaller"),
                                        ((64, 256, 0, 1), "window")])
def test_view_errors(args, match):
    with pytest.raises(ValueError, match=match):
        P.panorama_views(*args)


def test_colour_map_must_be_a_multiple_of_8():
    with pytest.raises(ValueError, match="multiple of 8"):
        P.paint_with_words_panorama({}, Image.new("RGB", (260, 128)), "a", device="cpu")
    with pytest.raises(ValueError, match="stride"):
        P.paint_with_words_panorama({}, Image.new("RGB", (256, 128)), "a", device="cpu", window=16, stride=17,
                                    preloaded_utils=(None,) * 5)


# ---- conditioning --------------------------------------------------------------------------------------------------
class _CountingEncoder(torch.nn.Module):
    def __init__(self, dim):
        super().__init__()
        self.inner, self.calls = RandomTextEncoder(dim), 0

    def forward(self, ids):
        self.calls += 1
        return self.inner(ids)


@pytest.mark.parametrize("circular", [False, True], ids=["flat", "circular"])
@pytest.mark.parametrize("chunks", [1, 2])
def test_window_conditioning_is_the_crops_conditioning(circular, chunks):
    cm = wide_color_map()
    s = SETTINGS["aurora"]
    ctx = dict(s["ctx"])
    ctx[(51, 193, 217)] = "mountains,0.4,7,3.0"                  # a regional seed and blur
    prompt = s["prompt"] + (" " + SETTINGS["cat_dog"]["prompt"]) * (4 if chunks > 1 else 0)   # 101 tokens
    tok = SimpleWordTokenizer()
    views = P.panorama_views(16, 32, 16, 8, circular)
    enc = _CountingEncoder(64)
    conds, unconds = PN.panorama_conditioning(enc, tok, "cpu", cm, ctx, prompt, "ugly", views, 16, chunks)
    assert enc.calls == 2 * chunks                                # the prompt and the uncond prompt, once each
    assert len(conds) == len(unconds) == len(views[0]) * len(views[1])
    pixels = np.array(cm)
    wrapped = 0
    for v, (y0, x0) in enumerate((y, x) for y in views[0] for x in views[1]):
        crop = np.roll(pixels, -8 * x0, axis=1)[8 * y0:8 * y0 + 128, :128]
        wrapped += 8 * x0 + 128 > cm.width
        assert np.array_equal(np.array(PN.window_crop(cm, y0, x0, 16)), crop)
        _, _, cond, uncond = _encode_text_color_inputs(RandomTextEncoder(64), tok, "cpu", Image.fromarray(crop),
                                                       dict(ctx), prompt, "ugly", max_prompt_chunks=chunks)
        for got, want in ((conds[v], cond), (unconds[v], uncond)):
            assert got.keys() == want.keys()
            for k in want:
                if torch.is_tensor(want[k]):
                    assert torch.equal(got[k], want[k]), (v, k)
                else:
                    assert got[k] == want[k], (v, k)
    assert wrapped == (1 if circular else 0)


def test_canvas_start_latents_are_the_whole_maps():
    cm = wide_color_map()
    ctx = dict(SETTINGS["aurora"]["ctx"])
    ctx[(7, 9, 182)] = "aurora,0.5,11"
    ctx[(51, 193, 217)] = "mountains,0.4,7,3.0"
    tok = SimpleWordTokenizer()
    extra_seeds, sep, _, _ = _encode_text_color_inputs(RandomTextEncoder(64), tok, "cpu", cm, dict(ctx),
                                                       SETTINGS["aurora"]["prompt"], "")
    assert len(extra_seeds) == 2
    want = initial_latents((1, 4, 16, 32), 5, extra_seeds, sep)
    got = PN.panorama_latents(cm, ctx, tok, 5)
    assert torch.equal(got, want) and not torch.equal(got, torch.randn(1, 4, 16, 32, generator=torch.manual_seed(5)))


# ---- the C entry points' argument checks ---------------------------------------------------------------------------
def test_window_entry_points_validate_before_any_cuda_call():
    L = _native.lib()
    buf = (ctypes.c_char * 4096)()
    p = (ctypes.addressof(buf) + 15) // 16 * 16

    def win_input(lat=p, first=0, n=2, window=16, dtype=1, h=16, w=48):
        # latents, scale, rows, n_rows, cols, n_cols, first, n, window, out, dtype, h, w, stream
        return L.pww_window_input(lat, p, p, 1, p, 5, first, n, window, p, dtype, h, w, None)
    assert win_input(lat=None) == -1
    assert win_input(window=17) == -1               # larger than the canvas
    assert win_input(first=4, n=2) == -1            # past the 5 windows
    assert win_input(dtype=2) == -2 and win_input(dtype=3) == -2

    def win_update(table, n_chunks, per_chunk=2, dtype=1, lat=p, n_cols=5):
        ptrs = (ctypes.c_void_p * len(table))(*table)
        return L.pww_window_update(ptrs, n_chunks, per_chunk, dtype, 2048, 1, 64, 4, p, 1, p, n_cols, 16, lat, p, 4,
                                   None, p, p, p, 16, 48, None)
    assert win_update([p] * 3, 3, dtype=2) == -2    # everything else valid: the dtype is what fails
    assert win_update([p] * 3, 3, lat=None) == -1
    assert win_update([p, None, p], 3) == -1        # a null chunk output
    assert win_update([p] * 2, 2) == -1             # 5 windows in chunks of 2 are 3 chunks
    assert win_update([p] * 65, 65, per_chunk=1, n_cols=65) == -1     # more than 64 chunks
    assert L.pww_window_update(None, 1, 5, 1, 2048, 1, 64, 4, p, 1, p, 5, 16, p, p, 4, None, p, p, p, 16, 48,
                               None) == -1


def _small_sampler_args(w=48, stride=8, window=16):
    views = P.panorama_views(16, w, window, stride)
    n = len(views[0]) * len(views[1])
    ctx = {"CONTEXT_TENSOR": torch.zeros(1, 77, 64)}
    sch = LMSDiscreteScheduler(**KW)
    sch.set_timesteps(2)
    return dict(unet=torch.nn.Linear(1, 1), scheduler=sch, cond_ctxs=[ctx] * n, uncond_ctxs=[ctx] * n,
                latents=torch.zeros(1, 4, 16, w), views=views, window=window, weight_function=WF)


def test_sampler_argument_errors():
    with pytest.raises(ValueError, match="at most 64"):
        PN.PanoramaSampler(**dict(_small_sampler_args(w=112, stride=1), view_batch_size=1))   # 97 chunks
    args = _small_sampler_args()
    with pytest.raises(ValueError, match="cond and"):
        PN.PanoramaSampler(**dict(args, cond_ctxs=args["cond_ctxs"][:-1]))
    with pytest.raises(ValueError, match="canvas"):
        PN.PanoramaSampler(**dict(args, latents=torch.zeros(2, 4, 16, 48)))
    with pytest.raises(ValueError, match="uncovered"):
        PN.PanoramaSampler(**dict(args, views=([0], [0, 8]), cond_ctxs=args["cond_ctxs"][:2],
                                  uncond_ctxs=args["uncond_ctxs"][:2]))
    with pytest.raises(ValueError, match="noise_seed"):
        sch = EulerAncestralDiscreteScheduler(**KW)
        sch.set_timesteps(2)
        PN.PanoramaSampler(**dict(args, scheduler=sch))
    s = PN.PanoramaSampler(**dict(args, view_batch_size=2))
    assert s.m == 2 and s._firsts == [0, 2, 4] and [x.shape[0] for x in s._unet_ins] == [4, 4, 2]
    # the last chunk's G_SIGMA: its one G value, then one uncond zero, from the step row's 2 G values and 2 zeros
    assert s._ctxs[2]["G_SIGMA"].data_ptr() == s._params[PN._G + 1:].data_ptr()
    assert s._ctxs[2]["G_SIGMA"].numel() == 2 and s._ctxs[0]["G_SIGMA"].numel() == 4


# ---- the reference loop's self-checks ------------------------------------------------------------------------------
class _WithNoise:
    def __init__(self, sch, noise):
        self._sch, self._noise, self._k = sch, noise, 0

    def __getattr__(self, name):
        return getattr(self._sch, name)

    def step(self, eps, t, x):
        out = self._sch.step(eps, t, x, noise=self._noise[self._k])
        self._k += 1
        return out


@pytest.mark.parametrize("name", ["lms", "dpmpp_2m", "euler_a"])
def test_one_window_canvas_is_the_reference_loop(name):
    cfg = UNetConfig.tiny()
    unet = build_unet(cfg, seed=0)
    s = SETTINGS["aurora"]
    try:
        oracle_loop.patch_with_oracle(unet)
        _, _, cond, uncond = _encode_text_color_inputs(RandomTextEncoder(64), SimpleWordTokenizer(), "cpu",
                                                       color_map_image("aurora", 128), dict(s["ctx"]), s["prompt"], "")
        steps = 3
        sch = SAMPLERS[name](**KW)
        sch.set_timesteps(steps)
        lat = torch.randn(1, 4, 16, 16, generator=torch.manual_seed(0)) * sch.init_noise_sigma
        noise = ancestral_noise([0], (4, 16, 16), steps) if name == "euler_a" else None
        got = panorama_loop.reference_panorama_loop(unet, sch, [cond], [uncond], lat, ([0], [0]), 16, WF, 7.5,
                                                    noise=noise)
        ref_sch = _WithNoise(sch, noise[:, 0]) if noise is not None else sch
        want = oracle_loop.reference_denoise_loop(unet, ref_sch, cond, uncond, lat, WF, 7.5)
    finally:
        cls = attention_modules(unet)[0].__class__
        if "__call__" in cls.__dict__:
            delattr(cls, "__call__")
    assert torch.equal(got, want)


class _ToyUNet:
    """A float64 stand-in whose output depends on the window's input and on its dict."""

    def __call__(self, x, t, encoder_hidden_states):
        c = encoder_hidden_states["CONTEXT_TENSOR"][0]
        out = torch.tanh(c[0].view(1, 4, 1, 1) * x + c[1].view(1, 4, 1, 1)) + 0.3 * torch.sin(x.roll(1, -1) * c[2, 0])

        class _Out:
            sample = out
        return _Out()


@pytest.mark.parametrize("prediction_type", ["epsilon", "v_prediction"])
@pytest.mark.parametrize("name", list(SAMPLERS))
@pytest.mark.parametrize("layout", [(12, 30, 8, 3, False), (12, 30, 8, 5, True), (8, 20, 8, 8, False)],
                         ids=["flush", "circular", "abutting"])
def test_average_then_step_is_step_then_average(name, prediction_type, layout):
    h, w, window, stride, circular = layout
    views = P.panorama_views(h, w, window, stride, circular)
    g = torch.Generator().manual_seed(1)
    V = len(views[0]) * len(views[1])
    conds = [{"CONTEXT_TENSOR": torch.randn(1, 3, 4, generator=g, dtype=torch.float64)} for _ in range(V)]
    unconds = [{"CONTEXT_TENSOR": torch.randn(1, 3, 4, generator=g, dtype=torch.float64)} for _ in range(V)]
    steps = 8
    sch = SAMPLERS[name](**KW, prediction_type=prediction_type)
    sch.set_timesteps(steps)
    lat = torch.randn(1, 4, h, w, generator=g, dtype=torch.float64) * float(sch.init_noise_sigma)
    noise = ancestral_noise([3], (4, h, w), steps).double() if name == "euler_a" else None
    a = panorama_loop.reference_panorama_loop(_ToyUNet(), sch, conds, unconds, lat, views, window, WF, 7.5, noise=noise)
    b = panorama_loop.canvas_step_loop(_ToyUNet(), sch, conds, unconds, lat, views, window, WF, 7.5, noise=noise)
    assert a.dtype == torch.float64 and torch.isfinite(a).all()
    assert (a - b).abs().max().item() <= 1e-12 * max(1.0, a.abs().max().item())
