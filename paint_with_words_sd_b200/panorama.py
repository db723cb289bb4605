"""Panoramas and wide canvases: MultiDiffusion (Bar-Tal et al. 2023; diffusers' `StableDiffusionPanoramaPipeline`)
over one colour map.

A canvas latent [1, 4, H, W] larger than the model's training size is covered with overlapping window x window crops.
Every step denoises each window with the UNet, and every canvas value takes the mean of the guided outputs of the
windows that cover it before the sampler's step form runs on the canvas.  Each window is conditioned on its own crop
of the colour map, so the colour map still says which words go where.

`panorama_views` lays out the windows, `panorama_conditioning` builds one cond / uncond dict per window,
`PanoramaSampler` runs the loop (per chunk of windows one `pww_window_input` launch and one UNet forward, then one
`pww_window_update` launch for the canvas, captured as one CUDA graph), and `paint_with_words_panorama` is the
public entry point.
"""
from __future__ import annotations

import ctypes
from typing import Callable, Dict, List, Optional, Sequence, Tuple

import numpy as np
import torch
from PIL import Image

from . import _native
from .conditioning import (_blur_image_mask, _encode_text_color_inputs, _extract_seed_and_sigma_from_context,
                           _image_context_seperator)
from .pipeline import (_BETA, _G, _SCALE, _T, PwWSampler, _dtype_code, _module_dtype, _result, _tools,
                       ancestral_noise, default_weight_function, initial_latents)
from .scheduler import (SIGMA_SCHEDULERS, EulerAncestralDiscreteScheduler, LMSDiscreteScheduler, history_length)
from .weight_function import probe_weight_function

MAX_WINDOW_CHUNKS = 64      # chunk pointers pww_window_update takes in its kernel parameters (csrc/sampler_window.cuh)


def _axis_starts(size: int, window: int, stride: int, wrap: bool) -> List[int]:
    if wrap:
        return list(range(0, size, stride))
    starts = list(range(0, size - window + 1, stride))
    if starts[-1] + window < size:          # the last window stops short of the edge: one more, flush with it
        starts.append(size - window)
    return starts


def panorama_views(height: int, width: int, window: int, stride: int = 8,
                   circular: bool = False) -> Tuple[List[int], List[int]]:
    """(row starts, column starts) of the windows over a [height, width] latent canvas; window v = iy * n_cols + ix
    has its origin at (rows[iy], cols[ix]).  On each axis the starts are 0, stride, 2 stride, ... while start + window
    <= size, plus one start at size - window if the last window stops short of the edge, so every value is covered.
    `circular` wraps the horizontal axis: column starts 0, stride, ... below `width`, a window reading canvas column
    (start + x) mod width.  ValueError for a stride outside 1..window or a canvas smaller than the window."""
    if window < 1:
        raise ValueError(f"window must be >= 1, got {window}")
    if not 1 <= stride <= window:
        raise ValueError(f"stride must be in 1..window ({window}), got {stride}")
    if height < window or width < window:
        raise ValueError(f"the {height}x{width} latent canvas is smaller than the {window}x{window} window")
    return _axis_starts(height, window, stride, False), _axis_starts(width, window, stride, circular)


def _check_views(rows: Sequence[int], cols: Sequence[int], window: int, height: int, width: int) -> None:
    """ValueError unless every window lies on the canvas (column starts may wrap) and every value is covered."""
    if not rows or not cols or window < 1 or window > min(height, width):
        raise ValueError(f"views: need row and column starts and a window of 1..{min(height, width)}, got "
                         f"{len(rows)} x {len(cols)} starts and window {window}")
    if any(not 0 <= r <= height - window for r in rows) or any(not 0 <= c < width for c in cols):
        raise ValueError(f"views: row starts must be in 0..{height - window} and column starts in 0..{width - 1}")
    cover_y, cover_x = np.zeros(height, bool), np.zeros(width, bool)
    for r in rows:
        cover_y[r:r + window] = True
    for c in cols:
        cover_x[np.arange(c, c + window) % width] = True
    if not (cover_y.all() and cover_x.all()):
        raise ValueError("views: the windows leave part of the canvas uncovered")


def window_crop(image: Image.Image, y0: int, x0: int, window: int) -> Image.Image:
    """The colour-map crop under the window at latent origin (y0, x0): `image.crop((8 x0, 8 y0, 8 (x0 + window),
    8 (y0 + window)))`, or for a window that wraps past the right edge the two pieces pasted side by side."""
    px, left, top = 8 * window, 8 * x0, 8 * y0
    if left + px <= image.width:
        return image.crop((left, top, left + px, top + px))
    first = image.width - left
    out = Image.new(image.mode, (px, px))
    out.paste(image.crop((left, top, image.width, top + px)), (0, 0))
    out.paste(image.crop((0, top, px - first, top + px)), (first, 0))
    return out


class _EncodeOnce:
    """A text encoder that keeps its output per token-id row: the windows share the prompt and the uncond prompt, so
    each is encoded once."""

    def __init__(self, text_encoder):
        self.text_encoder = text_encoder
        self._out: Dict[tuple, object] = {}

    def __call__(self, ids: torch.Tensor):
        key = (tuple(ids.shape), tuple(ids.flatten().tolist()))
        if key not in self._out:
            self._out[key] = self.text_encoder(ids)
        return self._out[key]


def panorama_conditioning(text_encoder, tokenizer, device, color_map_image: Image.Image, color_context: dict,
                          input_prompt: str, unconditional_input_prompt: str,
                          views: Tuple[Sequence[int], Sequence[int]], window: int,
                          max_prompt_chunks: int = 1) -> Tuple[List[dict], List[dict]]:
    """One (cond, uncond) dict per window, in window order: window v's is `_encode_text_color_inputs` of the colour-map
    crop under it (`window_crop`), weight maps, blur and packed maps included.  The prompts are encoded once."""
    encoder = _EncodeOnce(text_encoder)
    conds, unconds = [], []
    for y0 in views[0]:
        for x0 in views[1]:
            _, _, cond, uncond = _encode_text_color_inputs(
                encoder, tokenizer, device, window_crop(color_map_image, y0, x0, window), dict(color_context),
                input_prompt, unconditional_input_prompt, max_prompt_chunks=max_prompt_chunks)
            conds.append(cond)
            unconds.append(uncond)
    return conds, unconds


def panorama_latents(color_map_image: Image.Image, color_context: dict, tokenizer, seed: int) -> torch.Tensor:
    """The canvas's seeded start noise [1, 4, H/8, W/8] (before the scheduler's initial sigma): `initial_latents` of
    the whole colour map, so regional seeding ("label,strength,seed") works as in `paint_with_words`."""
    ctx, extra_seeds, extra_sigmas = _extract_seed_and_sigma_from_context(dict(color_context))
    seperated_word_contexts, width, height = _image_context_seperator(color_map_image, ctx, tokenizer)
    if extra_sigmas:
        seperated_word_contexts = _blur_image_mask(seperated_word_contexts, extra_sigmas)
    return initial_latents((1, 4, height // 8, width // 8), seed, extra_seeds, seperated_word_contexts)


class PanoramaSampler(PwWSampler):
    """MultiDiffusion denoising loop over one canvas on ONE GPU.

    `latents` is the canvas [1, 4, H, W]; `views` = (row starts, column starts) from `panorama_views` for `window`;
    `cond_ctxs` / `uncond_ctxs` hold one dict per window, in window order (`panorama_conditioning`).  Every window
    has the same `weight_function` and `guidance_scale`.  The windows are split into chunks of `view_batch_size`
    (a 2 * view_batch_size UNet batch with CFG; at most 64 chunks), each with its own merged context (weight-map
    stacks, K/V cache, scratch).  A step is, per chunk, `pww_window_input` and the UNet forward, then one
    `pww_window_update` that averages the windows' guided outputs at every canvas value and applies the sampler's
    step form on the canvas; `use_graph=True` captures it as one CUDA graph.

    The step rows, weight-function probing, graph capture, `step`, `run` and `restart` are PwWSampler's, with m =
    the chunk size.  Euler ancestral's step noise is `ancestral_noise([noise_seed], (4, H, W), n)`: one draw per
    canvas value.  Any sampler of `scheduler.py`, epsilon or v prediction, fp32 / fp16 / bf16 UNets; no ControlNets,
    adapters, masks, guidance rescale or attention recording."""

    def __init__(self, unet, scheduler, cond_ctxs: Sequence[dict], uncond_ctxs: Sequence[dict], latents: torch.Tensor,
                 views: Tuple[Sequence[int], Sequence[int]], window: int, weight_function: Callable,
                 guidance_scale: float = 7.5, noise_seed: Optional[int] = None, view_batch_size: int = 16,
                 use_graph: bool = True, timesteps=None):
        if not isinstance(scheduler, SIGMA_SCHEDULERS):
            raise TypeError(f"PanoramaSampler does not support {type(scheduler).__name__}; use one of "
                            + ", ".join(c.__name__ for c in SIGMA_SCHEDULERS))
        if latents.dim() != 4 or tuple(latents.shape[:2]) != (1, 4):
            raise ValueError(f"latents must be the canvas [1, 4, H, W], got {tuple(latents.shape)}")
        if getattr(unet, "in_channels", 4) != 4:
            raise ValueError(f"a panorama needs a 4-channel UNet, got in_channels = {unet.in_channels}")
        height, width = (int(s) for s in latents.shape[-2:])
        rows, cols = [int(r) for r in views[0]], [int(c) for c in views[1]]
        _check_views(rows, cols, int(window), height, width)
        V = len(rows) * len(cols)
        if len(cond_ctxs) != V or len(uncond_ctxs) != V:
            raise ValueError(f"{V} windows need {V} cond and {V} uncond dicts, got {len(cond_ctxs)} and "
                             f"{len(uncond_ctxs)}")
        if view_batch_size < 1:
            raise ValueError(f"view_batch_size must be >= 1, got {view_batch_size}")
        n = min(int(view_batch_size), V)
        firsts = list(range(0, V, n))
        if len(firsts) > MAX_WINDOW_CHUNKS:
            raise ValueError(f"{V} windows at view_batch_size {view_batch_size} make {len(firsts)} chunks; at most "
                             f"{MAX_WINDOW_CHUNKS}: raise view_batch_size or the stride")
        self.unet, self.scheduler, self.m = unet, scheduler, n
        self.device = latents.device
        self.weight_function, self.guidance_scale = weight_function, float(guidance_scale)
        self.window, self.views = int(window), (rows, cols)
        self.timesteps = list((scheduler.timesteps if timesteps is None else timesteps).tolist())
        self.latents = latents.to(torch.float32, memory_format=torch.contiguous_format, copy=True)
        self.use_graph = use_graph and latents.is_cuda
        self._fns, self._probed = [weight_function] * n, [probe_weight_function(weight_function, 1.0)] * n
        self._blend, self._nets, self._rec_levels, self.record_attention = None, [], [], False
        self._graphs, self._kv_graph, self._step_no = {}, None, 0
        self._active_sets = [()] * len(self.timesteps)
        dev = self.device
        self._hist_len = history_length(scheduler)
        self._form = _G + 2 * n
        self._rows = self._build_rows().to(dev)
        self._params = torch.zeros(self._rows.shape[1], dtype=torch.float32, device=dev)
        self._derivs = torch.zeros((self._hist_len,) + tuple(self.latents.shape), dtype=torch.float32, device=dev)
        self._gscale = torch.tensor([self.guidance_scale], dtype=torch.float32, device=dev)
        self._starts = (torch.tensor(rows, dtype=torch.int32, device=dev), torch.tensor(cols, dtype=torch.int32, device=dev))
        self._noise = None
        if isinstance(scheduler, EulerAncestralDiscreteScheduler):
            if not isinstance(noise_seed, (int, np.integer)):
                raise ValueError(f"{type(scheduler).__name__} draws noise every step: pass noise_seed (one int)")
            self._noise = ancestral_noise([noise_seed], (4, height, width), len(self.timesteps)).to(dev)
        # per chunk: its first window, its merged context and its UNet input [2k, 4, window, window]
        self._firsts, self._ctxs, self._unet_ins = firsts, [], []
        for first in firsts:
            k = min(n, V - first)
            ctx = self._merge_contexts(cond_ctxs[first:first + k], uncond_ctxs[first:first + k])
            # the step row holds n equal G values (one weight function), then n zeros: the k before the zeros and k
            # zeros are this chunk's [2k] G_SIGMA
            ctx["G_SIGMA"] = self._params[_G + n - k:_G + n + k]
            self._ctxs.append(ctx)
            self._unet_ins.append(torch.empty((2 * k, 4, self.window, self.window), dtype=_module_dtype(unet),
                                              device=dev))

    def _step_body(self, active: tuple = ()):
        L = _native.lib()
        stream = torch.cuda.current_stream(self.device).cuda_stream
        p, (h, w), win = self._params, self.latents.shape[-2:], self.window
        rows, cols = self._starts
        t = p[_T:_T + 1]
        outs = []
        for first, ctx, x in zip(self._firsts, self._ctxs, self._unet_ins):
            k = x.shape[0] // 2
            _native.check(L.pww_window_input(self.latents.data_ptr(), p[_SCALE:].data_ptr(), rows.data_ptr(),
                                             rows.numel(), cols.data_ptr(), cols.numel(), first, k, win, x.data_ptr(),
                                             _dtype_code(x.dtype), h, w, stream), "pww_window_input")
            eps = self.unet(x, t, encoder_hidden_states=ctx).sample
            if tuple(eps.shape) != (2 * k, 4, win, win) or eps.device != self.device:
                raise ValueError(f"the UNet returned {tuple(eps.shape)} on {eps.device}; expected {(2 * k, 4, win, win)}")
            outs.append(eps)
        if len({(e.dtype, e.stride()) for e in outs}) != 1:
            raise ValueError("the UNet's chunk outputs differ in dtype or layout: "
                             + ", ".join(f"{e.dtype} {e.stride()}" for e in outs))
        # every chunk's output read in place: the pointer table goes into the kernel parameters (and a captured graph)
        table = (ctypes.c_void_p * len(outs))(*[e.data_ptr() for e in outs])
        e0 = outs[0]
        _native.check(L.pww_window_update(table, len(outs), self.m, _dtype_code(e0.dtype), *e0.stride(),
                                          rows.data_ptr(), rows.numel(), cols.data_ptr(), cols.numel(), win,
                                          self.latents.data_ptr(), self._derivs.data_ptr(), self._hist_len,
                                          None if self._noise is None else self._noise.data_ptr(),
                                          self._gscale.data_ptr(), p[_BETA:].data_ptr(), p[self._form:].data_ptr(),
                                          h, w, stream), "pww_window_update")
        _native.launch_count += len(outs) + 1

    def _set_step_scalars(self, i: int, step_index: int):
        self._params.copy_(self._rows[i])
        for ctx in self._ctxs:
            ctx["SIGMA"] = self.scheduler.sigmas[step_index]

    def device_inputs(self) -> Dict[str, torch.Tensor]:
        """The canvas latents (new values may be copied into them between graph replays)."""
        return {"latents": self.latents}


@torch.no_grad()
def paint_with_words_panorama(
    color_context: Dict[Tuple[int, int, int], str] = {},
    color_map_image: Optional[Image.Image] = None,
    input_prompt: str = "",
    num_inference_steps: int = 30,
    guidance_scale: float = 7.5,
    seed: int = 0,
    scheduler_type=LMSDiscreteScheduler,
    device: str = "cuda:0",
    weight_function: Callable = default_weight_function,
    local_model_path: Optional[str] = None,
    hf_model_path: Optional[str] = "synthetic:sd15",
    preloaded_utils: Optional[Tuple] = None,
    unconditional_input_prompt: str = "",
    model_token: Optional[str] = None,
    return_latents: bool = False,
    max_prompt_chunks: int = 1,
    torch_dtype: Optional[torch.dtype] = None,
    prediction_type: Optional[str] = None,
    window: Optional[int] = None,
    stride: int = 8,
    circular_padding: bool = False,
    view_batch_size: int = 16,
):
    """A panorama or any canvas larger than the model's training size, laid out by one colour map (MultiDiffusion).
    Returns one PIL image of the colour map's size, or the canvas latents [1, 4, H/8, W/8] with `return_latents`.

    The colour map's width and height must be multiples of 8.  `window` (latent pixels) defaults to the UNet's
    `config.sample_size` (64 for SD1.5, 96 for SD2.x), `stride` to 8; `circular_padding` wraps the horizontal axis
    (360-degree panoramas); see `panorama_views`.  Each window is conditioned on its crop of the colour map, and the
    start latents are the whole colour map's (`initial_latents`, regional seeds included).  `view_batch_size` windows
    share one UNet batch.  The other arguments are `paint_with_words`'s."""
    if color_map_image is None:
        raise ValueError("paint_with_words_panorama needs a color_map_image")
    width, height = color_map_image.size
    if width % 8 or height % 8:
        raise ValueError(f"the colour map's size {width}x{height} must be a multiple of 8 on both axes")
    tools = _tools(preloaded_utils, device, scheduler_type, local_model_path, hf_model_path, model_token, torch_dtype,
                   prediction_type)
    vae, unet, text_encoder, tokenizer, scheduler = tools
    window = int(unet.config.sample_size) if window is None else int(window)
    views = panorama_views(height // 8, width // 8, window, stride, circular_padding)
    scheduler.set_timesteps(num_inference_steps)
    conds, unconds = panorama_conditioning(text_encoder, tokenizer, device, color_map_image, color_context,
                                           input_prompt, unconditional_input_prompt, views, window, max_prompt_chunks)
    latents = panorama_latents(color_map_image, color_context, tokenizer, seed).to(device) * scheduler.init_noise_sigma
    sampler = PanoramaSampler(unet, scheduler, conds, unconds, latents, views, window, weight_function, guidance_scale,
                              noise_seed=seed, view_batch_size=view_batch_size)
    return _result(vae, sampler.run(), return_latents)
