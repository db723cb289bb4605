"""Public API: `paint_with_words()`, `paint_with_words_inpaint()`, `pww_load_tools()` -- same keyword
arguments, defaults and return type as the reference (paint_with_words/paint_with_words.py:128-204,
391-510; paint_with_words_inpaint.py:137-270) -- plus `PwWSampler`, the GPU-first engine behind them, and
`paint_with_words_batch()`, which makes many differently configured images in shared samplers.

What is different underneath (results equal within the stated fp16 tolerance):
  * the attention of every UNet block runs in libpww_b200.so (see attention.py);
  * cond and uncond are ONE batch-2 UNet forward with per-image bias enable and per-image score
    statistic instead of two batch-1 forwards (paint_with_words.py:483-499);
  * the whole step (UNet input, UNet, CFG combine + sampler update as two native launches) is captured in a CUDA
    graph; sigma, G(sigma) and the sampler's step-form coefficients are device scalars refreshed by one tiny copy, so
    a replay does no host math;
  * K/V of the text context are step-invariant, so the context tensors are staged once per image.
"""
from __future__ import annotations

import dataclasses
import inspect
import math
from typing import Callable, Dict, List, Optional, Sequence, Tuple, Union

import numpy as np
import torch
import torch.nn.functional as F
from PIL import Image

from . import attention as _attention
from .conditioning import (MAX_RECORDED_REGIONS, RATIOS, REGION_COUNT_KEY, REGION_INDEX_KEY,
                           _encode_text_color_inputs, _extract_seed_and_sigma_from_context, _get_binary_mask,
                           _rgb_of, always_round, pack_weight_map, packed_key)
from . import _native, fused_ops
from .scheduler import (SIGMA_SCHEDULERS, EulerAncestralDiscreteScheduler, LMSDiscreteScheduler, history_length,
                        step_form)
from .synthetic import IdentityVAE, RandomTextEncoder, SimpleWordTokenizer
from .unet import UNet2DConditionModel, UNetConfig, build_unet, combine_control_residuals
from .weight_function import STAT_MAX, UnsupportedWeightFunction, g_of_sigma, probe_weight_function


def default_weight_function(w, sigma, qk):
    """paint_with_words.py:402-405."""
    return 0.1 * w * math.log(sigma + 1) * qk.max()


def _zero_weight_function(w, sigma, qk):
    """The uncond branch's `lambda w, sigma, qk: 0.0` (paint_with_words.py:493)."""
    return 0.0


_SYNTHETIC_CONFIGS = {
    "synthetic:sd15": UNetConfig.sd15,
    "synthetic:sd15-inpaint": UNetConfig.sd15_inpaint,
    "synthetic:sd21": UNetConfig.sd21,
    "synthetic:tiny": UNetConfig.tiny,
    "synthetic:tiny-inpaint": lambda: UNetConfig.tiny(in_channels=9),
}


def pww_load_tools(device: str = "cuda:0", scheduler_type=LMSDiscreteScheduler,
                   local_model_path: Optional[str] = None, hf_model_path: Optional[str] = None,
                   model_token: Optional[str] = None, seed: int = 0, torch_dtype: Optional[torch.dtype] = None):
    """paint_with_words.py:128-204: returns (vae, unet, text_encoder, tokenizer, scheduler) with the
    attention of `unet` patched.  `"synthetic:<sd15|sd15-inpaint|sd21|tiny>"` model paths build seeded
    random-weight stand-ins (no weights or network exist in this environment); any other path is
    loaded with diffusers/transformers when those are installed.
    `torch_dtype`: the UNet's (and VAE's) dtype; None keeps the reference's rule (fp16, fp32 on mps), and
    torch.bfloat16 runs every native kernel in bf16."""
    assert local_model_path or hf_model_path, "either local_model_path or hf_model_path must be provided"
    model_path = local_model_path if local_model_path is not None else hf_model_path
    dtype = torch_dtype if torch_dtype is not None else (torch.float16 if device != "mps" else torch.float32)
    if model_path in _SYNTHETIC_CONFIGS:
        cfg = _SYNTHETIC_CONFIGS[model_path]()
        unet = build_unet(cfg, seed=seed, dtype=dtype, device=device)
        text_encoder = RandomTextEncoder(cfg.cross_attention_dim).to(device)
        tokenizer, vae = SimpleWordTokenizer(), IdentityVAE().to(device)
    else:
        try:
            from diffusers import AutoencoderKL, UNet2DConditionModel as _HFUNet
            from transformers import CLIPTextModel, CLIPTokenizer
        except ImportError as e:
            raise ImportError(f"loading '{model_path}' needs diffusers + transformers, which are not installed; "
                              "use a 'synthetic:*' model path or pass preloaded_utils") from e
        local_only = local_model_path is not None
        vae = AutoencoderKL.from_pretrained(model_path, subfolder="vae", torch_dtype=dtype,
                                            local_files_only=local_only).to(device)
        tokenizer = CLIPTokenizer.from_pretrained(model_path, subfolder="tokenizer")
        text_encoder = CLIPTextModel.from_pretrained(model_path, subfolder="text_encoder").to(device)
        unet = _HFUNet.from_pretrained(model_path, subfolder="unet", torch_dtype=dtype,
                                       local_files_only=local_only).to(device)
    _attention.patch_unet(unet)
    scheduler = scheduler_type(beta_start=0.00085, beta_end=0.012, beta_schedule="scaled_linear",
                               num_train_timesteps=1000)
    return vae, unet, text_encoder, tokenizer, scheduler


def _dtype_code(dtype) -> int:
    """The C ABI's dtype code; -1 (rejected by the kernels as unsupported) for anything but fp32 / fp16 / bf16."""
    return {torch.float32: _native.PWW_DTYPE_F32, torch.float16: _native.PWW_DTYPE_F16,
            torch.bfloat16: _native.PWW_DTYPE_BF16}.get(dtype, -1)


def _module_dtype(module, default=torch.float32):
    p = next(iter(module.parameters()), None) if hasattr(module, "parameters") else None
    return p.dtype if p is not None else default


def _pil_from_latents(vae, latents):
    """paint_with_words.py:48-57.  (The reference runs under torch.autocast; here the VAE gets its own dtype.)"""
    image = vae.decode((1 / 0.18215 * latents.clone()).to(_module_dtype(vae, latents.dtype))).sample
    image = (image / 2 + 0.5).clamp(0, 1).detach().cpu().permute(0, 2, 3, 1).float().numpy()
    return [Image.fromarray(a) for a in (image * 255).round().astype("uint8")]


def preprocess(image):
    """paint_with_words.py:28-35."""
    w, h = image.size
    w, h = w - w % 32, h - h % 32
    arr = np.array(image.resize((w, h), resample=Image.LANCZOS)).astype(np.float32) / 255.0
    return 2.0 * torch.from_numpy(arr[None].transpose(0, 3, 1, 2)) - 1.0


def initial_latents(latent_size, seed: int, extra_seeds: Dict[int, int], seperated_word_contexts) -> torch.Tensor:
    """paint_with_words.py:445-455: host-side seeded noise, optionally re-seeded per region."""
    latents = torch.randn(latent_size, generator=torch.manual_seed(seed))
    if len(extra_seeds) > 0:
        print("Use region based seeding: ", extra_seeds)
        per_seed = [torch.randn(latent_size, generator=torch.manual_seed(s)) for s in extra_seeds.values()]
        masks = _get_binary_mask(seperated_word_contexts, extra_seeds, dtype=latents[0].dtype, size=latent_size[-2:])
        foreground = (sum(masks) > 0).squeeze()
        mixed = sum(l * m for l, m in zip(per_seed, masks))
        latents[:, :, foreground] = mixed[:, :, foreground]
    return latents


# ---------------------------------------------------------------------------------------------
# the engine
# ---------------------------------------------------------------------------------------------
def ancestral_noise(seeds: Sequence[int], shape: Tuple[int, ...], n: int) -> torch.Tensor:
    """[n, m, *shape] fp32: image i's rows are draws 1..n of `torch.Generator().manual_seed(seeds[i])` on the CPU, each
    `shape`-sized (draw 0 is that seed's initial noise), as a diffusers pipeline given `generator=torch.manual_seed(seed)`
    draws them.  Per image, so batching and sharding do not change which noise an image gets."""
    per_image = []
    for s in seeds:
        g = torch.Generator().manual_seed(int(s))
        torch.randn(shape, generator=g)
        per_image.append(torch.stack([torch.randn(shape, generator=g) for _ in range(n)]))
    return torch.stack(per_image, 1)


def _per_image(value, m: int, name: str, is_one) -> list:
    """One setting for every image, or a sequence of exactly m settings."""
    if is_one(value):
        return [value] * m
    vals = list(value)
    if len(vals) != m or not all(is_one(v) for v in vals):
        raise ValueError(f"{name} must be one value or a sequence of {m} (one per image)")
    return vals


# guess mode scales ControlNet residual k (0..12, the mid residual last) by 0.825 ** (12 - k) (hook_pww.py:132)
GUESS_MODE_DECAY = 0.825


def control_scales(conditioning_scales: Sequence[float], guess_mode: bool, levels: int = 13) -> torch.Tensor:
    """CONTROL_SCALES for m images with these ControlNet weights: fp32 [levels, rows].  Plain: rows = 2m, column i and
    column m + i both hold weight_i (the cond and uncond image share the residual's weight).  Guess mode: rows = m
    (only the cond half gets residuals), entry [k, i] = weight_i * 0.825 ** (levels - 1 - k)."""
    w = torch.tensor([float(s) for s in conditioning_scales], dtype=torch.float64)
    if guess_mode:
        decay = torch.tensor([GUESS_MODE_DECAY ** float(levels - 1 - k) for k in range(levels)], dtype=torch.float64)
        return (decay[:, None] * w[None, :]).to(torch.float32)
    return torch.cat([w, w]).to(torch.float32)[None, :].repeat(levels, 1)


def control_step_active(i: int, n: int, start: float, end: float) -> bool:
    """Is the ControlNet applied at step i (0-based) of n?  hook_pww.py:23-26: iff start <= i / n <= end."""
    return start <= i / n <= end


MAX_CONTROLNET_UNITS = 10      # the reference extension's "Multi ControlNet: Max models amount"


def _control_units(controlnet, control_image, conditioning_scale, guess_mode, start, end) -> tuple:
    """The ControlNet arguments as per-unit lists (nets, images, weights, guesses, starts, ends), for one ControlNet or
    a list of them.  One ControlNetModel is one unit with the arguments as they are.  A list of U (1..10) units takes
    `control_image` as a list of U entries (each one tensor or one per image), `controlnet_conditioning_scale` as one
    float or U entries (each one float or one per image), and `guess_mode` and the window each as one value or U values;
    lists are indexed by unit first.  The per-unit lists, passed in again, come out unchanged (`_control_arguments`
    hands them to PwWSampler)."""
    if not isinstance(controlnet, (list, tuple)):
        return [controlnet], [control_image], [conditioning_scale], [bool(guess_mode)], [start], [end]
    U = len(controlnet)
    if not 1 <= U <= MAX_CONTROLNET_UNITS:
        raise ValueError(f"controlnet: a list of 1 to {MAX_CONTROLNET_UNITS} ControlNets, got {U}")
    if not isinstance(control_image, (list, tuple)) or len(control_image) != U:
        got = f"{len(control_image)} entries" if isinstance(control_image, (list, tuple)) else type(control_image).__name__
        raise ValueError(f"control_image must be a list of {U} entries, one per ControlNet (each one [1, 3, H, W] "
                         f"tensor or one per image), got {got}")

    def per_unit(value, name, is_one):
        if is_one(value):
            return [value] * U
        if not isinstance(value, (list, tuple)) or len(value) != U:
            raise ValueError(f"{name} must be one value or a list of {U} (one per ControlNet), got {value!r}")
        return list(value)
    number = lambda v: isinstance(v, (int, float)) and not isinstance(v, bool)   # noqa: E731
    weights = per_unit(conditioning_scale, "controlnet_conditioning_scale", number)
    guesses = per_unit(guess_mode, "guess_mode", lambda v: isinstance(v, (bool, np.bool_)))
    starts = per_unit(start, "control_guidance_start", number)
    ends = per_unit(end, "control_guidance_end", number)
    return list(controlnet), list(control_image), weights, [bool(g) for g in guesses], starts, ends


def control_image_tensor(image: Image.Image) -> torch.Tensor:
    """A hint image as the ControlNet takes it: HWC RGB -> float / 255 -> [1, 3, H, W] in [0, 1] (no [-1, 1] remap)."""
    arr = np.asarray(image.convert("RGB"), dtype=np.float32) / 255.0
    return torch.from_numpy(arr.transpose(2, 0, 1).copy())[None]


# Columns of a step row.  PwWSampler tabulates one row per step at set-up (`_rows`) and a step copies its row into
# `_params` (one D2D copy), so a captured graph reads new values through the same device pointers:
_SIGMA = 0    # sigma
_SCALE = 1    # 1/sqrt(sigma^2 + 1): pww_sampler_input's `scale`
_T = 2        # the timestep: the UNet's and the ControlNet's `timestep`
_BETA = 3     # beta0..beta3: pww_sampler_update's `beta`
_G = 7        # G_0(sigma) .. G_{m-1}(sigma), then m zeros for the uncond images: the attention's G_SIGMA
# after them, at _G + 2m, scheduler.FORM_COLUMNS (alpha, a, b, gamma, slot, row): pww_sampler_update's `form`


class PwWSampler:
    """Denoising loop for a group of images on ONE GPU (paint_with_words.py:471-506 semantics per image).

    Each image i has a cond context dict, an uncond context dict and latents; a step runs one UNet
    forward over the batch [cond_0..cond_{m-1}, uncond_0..uncond_{m-1}], the CFG combine and the sampler update.
    `use_graph=True` captures the step in a CUDA graph.

    `scheduler` is an LMS, Euler, Euler ancestral or DPM++ 2M scheduler of `scheduler.py` (any other class raises
    TypeError).  Every sampler is one linear step form per image (`scheduler.step_form`), tabulated for every step at
    set-up.  The ancestral sampler needs `noise_seed` (one int, or m ints): image i's step noise is
    `ancestral_noise([seed_i], ...)`; the other samplers ignore it.

    `weight_function` is one callable for every image or a sequence of m callables, one per image, and `guidance_scale`
    one float or m floats: images made with different settings share the sampler, and every cross-attention call is
    still one launch (per-image statistic kind and G(sigma) on the device).  An identically-zero function leaves its
    image unbiased.

    ControlNet (`controlnet`, a `controlnet.ControlNetModel` built for the UNet's config): `control_image` is one
    [1, 3, 8h, 8w] tensor in [0, 1] per image (one tensor for every image, or m), `controlnet_conditioning_scale` one
    weight or m.  At set-up every image's hint is embedded once (it does not depend on the step) and the weights become
    the UNet's CONTROL_SCALES table.  A step then runs the ControlNet on the first 4 channels of the UNet input with the
    plain text context (the reference builds the PwW dict only afterwards, hook_pww.py:113-149), and the UNet adds its
    13 residuals in one native launch.  `guess_mode`: the ControlNet sees only the m cond images, residual k is weighted
    by 0.825 ** (12 - k) and only the cond half gets them (hook_pww.py:28-61, 128-132).  Step i of n is controlled iff
    `control_guidance_start <= i / n <= control_guidance_end`; the other steps replay a second graph without the
    ControlNet, captured only when some step needs it.

    Multi-ControlNet (the extension's control units): `controlnet` a list of 1..10 ControlNetModels, `control_image` a
    list with one entry per unit (each one tensor or m), and `controlnet_conditioning_scale`, `guess_mode` and the window
    each one value or one per unit (a unit's weight may again be m floats); one ControlNet is a list of one.  The units
    active at a step run in unit order.  With one active unit, the UNet's inject scales its residuals as above.  With
    two or more, their residuals are scaled (0.825 ** (12 - k) for a unit in guess mode) and summed level by level in
    ONE native combine, and the UNet adds the sum.  If any unit is in guess mode, every unit runs on the m cond rows and
    only the cond half gets residuals (hook_pww.py:39-53, 199).  Each set of active units over the run has its own
    captured graph.

    T2I-Adapters (`adapter.T2IAdapter`, from `pww_load_adapter`) are control units too: an entry of `controlnet` may
    be one, with its `control_image`, weight, guess mode and window taken exactly as a ControlNet unit's.  At set-up
    every adapter runs once on its hints (its features do not depend on the step), a feature is resized (nearest) where
    its level's size differs from the UNet's, and for every active set the active adapters' features, scaled (weight *
    (0.25, 0.62, 0.825, 1.0) per level in guess mode) and summed in unit order, are stored at fixed addresses.  A step
    hands that sum to the UNet (`down_intrablock_additional_residuals`), which adds it inside the residual epilogue of
    each encoder level's last layer: an adapter costs no extra launch per step.  ControlNet residuals reach the skips
    after the encoder has run, so a skip carries its adapter feature and then its ControlNet residual.

    `record_attention=True` records, inside the UNet's cross-attention launches (`pww_xattn_fused_rec_*`), the softmax
    mass every painted region's tokens receive from each pixel of each cond image, biased or not; `attention_maps()`
    returns it per image as [R, h, w] maps.  The accumulators are zeroed at set-up and by `restart()`.  The latents are
    the same bits as without recording.  The ControlNets' cross-attention is not recorded.
    """

    def __init__(self, unet, scheduler: LMSDiscreteScheduler, cond_ctxs: Sequence[dict], uncond_ctxs: Sequence[dict],
                 latents: torch.Tensor, weight_function: Union[Callable, Sequence[Callable]],
                 guidance_scale: Union[float, Sequence[float]] = 7.5,
                 extra_input: Optional[torch.Tensor] = None, use_graph: bool = True, timesteps=None,
                 noise_seed: Union[None, int, Sequence[int]] = None, controlnet=None,
                 control_image: Union[None, torch.Tensor, Sequence[torch.Tensor]] = None,
                 controlnet_conditioning_scale: Union[float, Sequence[float]] = 1.0, guess_mode: bool = False,
                 control_guidance_start: float = 0.0, control_guidance_end: float = 1.0,
                 record_attention: bool = False):
        if not isinstance(scheduler, SIGMA_SCHEDULERS):
            raise TypeError(f"PwWSampler does not support {type(scheduler).__name__}; use one of "
                            + ", ".join(c.__name__ for c in SIGMA_SCHEDULERS))
        self.unet, self.scheduler = unet, scheduler
        self.m = len(cond_ctxs)
        self.device = latents.device
        self.weight_function = weight_function
        self.guidance_scale = (float(guidance_scale) if isinstance(guidance_scale, (int, float))
                               else [float(g) for g in guidance_scale])
        self._fns = _per_image(weight_function, self.m, "weight_function", callable)
        scales = _per_image(self.guidance_scale, self.m, "guidance_scale", lambda g: isinstance(g, float))
        self.timesteps = list((scheduler.timesteps if timesteps is None else timesteps).tolist())
        # the sampler kernels index latents [m,4,h,w] and extra_input [m,5,h,w] as contiguous fp32 buffers: a private
        # contiguous copy, whatever the caller's layout, and shapes checked against the m images
        if latents.dim() != 4 or tuple(latents.shape[:2]) != (self.m, 4):
            raise ValueError(f"latents must be [{self.m}, 4, h, w] (one per image), got {tuple(latents.shape)}")
        self.latents = latents.to(torch.float32, memory_format=torch.contiguous_format, copy=True)
        if extra_input is not None and tuple(extra_input.shape) != (self.m, 5) + tuple(latents.shape[2:]):
            raise ValueError(f"extra_input must be [{self.m}, 5, {latents.shape[2]}, {latents.shape[3]}] (mask + masked-"
                             f"image latents per image), got {tuple(extra_input.shape)}")
        self.extra_input = (None if extra_input is None else     # inpaint: [m,5,h,w] (mask + masked-image latents)
                            extra_input.to(self.device, torch.float32, memory_format=torch.contiguous_format))
        self.use_graph = use_graph and latents.is_cuda
        self._graphs = {}                  # "the step runs the ControlNet" -> (captured step, its native launches)
        self._kv_graph = None
        self._probed = []
        for i, f in enumerate(self._fns):
            try:
                self._probed.append(probe_weight_function(f, 1.0))
            except UnsupportedWeightFunction as e:
                if callable(weight_function):
                    raise
                raise UnsupportedWeightFunction(f"weight_function of image {i}: {e}") from e
        self._ctx = self._merge_contexts(cond_ctxs, uncond_ctxs)
        dev = self.device
        # the step rows (column layout above); `_table` is the columns up to the images' G, without the uncond zeros
        m = self.m
        self._hist_len = history_length(scheduler)
        self._form = _G + 2 * m                # the step form's first column
        self._rows = self._build_rows().to(dev)
        self._table = self._rows[:, :_G + m]
        self._params = torch.zeros(self._rows.shape[1], dtype=torch.float32, device=dev)
        self._derivs = torch.zeros((self._hist_len,) + tuple(self.latents.shape), dtype=torch.float32, device=dev)
        self._ctx["G_SIGMA"] = self._params[_G:self._form]
        self._gscale = torch.tensor(scales, dtype=torch.float32, device=dev).view(m, 1, 1, 1)
        self._noise = None
        if isinstance(scheduler, EulerAncestralDiscreteScheduler):
            if noise_seed is None:
                raise ValueError(f"{type(scheduler).__name__} draws noise every step: pass noise_seed (one int or {m})")
            seeds = _per_image(noise_seed, m, "noise_seed", lambda v: isinstance(v, (int, np.integer)))
            self._noise = ancestral_noise(seeds, tuple(self.latents.shape[1:]), len(self.timesteps)).to(dev)
        channels = 4 + (0 if self.extra_input is None else int(self.extra_input.shape[1]))
        self._unet_in = torch.empty((2 * m, channels) + tuple(self.latents.shape[2:]), dtype=_module_dtype(unet),
                                    device=dev)
        self._step_no = 0
        self.controlnet = controlnet
        self.guess_mode = bool(guess_mode)
        self._nets: List = []              # the control units (ControlNets and T2I-Adapters), in unit order
        self._is_adapter: List[bool] = []
        self._combine_scales: Dict[tuple, torch.Tensor] = {}         # active set -> its ControlNets' scale tables
        self._adapter_sums: Dict[tuple, List[torch.Tensor]] = {}     # active set -> its adapters' summed features
        self._active_sets = [()] * len(self.timesteps)      # step i -> which units run (one bool per unit)
        self._control_active = [False] * len(self.timesteps)
        if controlnet is None:
            if control_image is not None:
                raise ValueError("control_image is given but controlnet is None")
        else:
            self._set_up_control(*_control_units(controlnet, control_image, controlnet_conditioning_scale, guess_mode,
                                                 control_guidance_start, control_guidance_end))
        self.record_attention = bool(record_attention)
        self._rec_levels: List[tuple] = []     # (N, h_r, w_r, accumulator [m, H, N, 16]) per cross-attention level
        if self.record_attention:
            self._set_up_recording(cond_ctxs)

    def _set_up_recording(self, conds):
        """record_attention: the cond images' token -> region rows, and one zeroed fp32 [m, H_l, N_l, 16] accumulator per
        UNet level, at fixed addresses (captured graphs add into them).  Level l has N_l = h_r * w_r query rows, the grid
        the weight-map builder uses at ratio 8 * 2^l, and the UNet config's head count of that level."""
        m, dev = self.m, self.device
        rows = [c.get(REGION_INDEX_KEY) for c in conds]
        if any(r is None for r in rows):
            raise ValueError(f"record_attention needs every cond dict's {REGION_INDEX_KEY} (set by the conditioning "
                             f"builder for at most {MAX_RECORDED_REGIONS} regions)")
        self._region_counts = [int(c[REGION_COUNT_KEY]) for c in conds]
        ridx = torch.stack([r.to(torch.int8) for r in rows], 0).contiguous().to(dev)
        rec_index = torch.tensor(list(range(m)) + [-1] * m, dtype=torch.int32, device=dev)   # only the cond rows
        cfg = getattr(self.unet, "config", None)
        heads = getattr(cfg, "attention_heads", getattr(cfg, "attention_head_dim", None))
        channels = getattr(cfg, "block_out_channels", None)
        if heads is None or channels is None:
            raise TypeError(f"record_attention needs the UNet config's block_out_channels and attention heads "
                            f"({type(self.unet).__name__} has none)")
        heads = list(heads) if isinstance(heads, (list, tuple)) else [int(heads)] * len(channels)
        h, w = self.latents.shape[-2:]
        for lvl, r in enumerate(RATIOS[:len(channels)]):
            hr, wr = always_round(8 * h / r), always_round(8 * w / r)
            self._rec_levels.append((hr * wr, hr, wr, torch.zeros((m, int(heads[lvl]), hr * wr, MAX_RECORDED_REGIONS),
                                                                   dtype=torch.float32, device=dev)))
        self._ctx[_attention.RECORD_KEY] = {n: (ridx, rec_index, acc) for n, _, _, acc in self._rec_levels}
        # every cross-attention module (a transformer block's attn2) is called once per UNet forward
        self._rec_calls = sum(1 for name, _ in self.unet.named_modules() if name.split(".")[-1] == "attn2")

    def attention_maps(self) -> List[torch.Tensor]:
        """record_attention: per cond image, fp32 [R, h, w] on the CPU at latent resolution, R = its regions.  Map r is
        the mean, over every recorded (step, cross-attention call, head), of the softmax mass the tokens of region r's
        label receive, upsampled bilinearly (align_corners=False) from the call's grid to the latent grid."""
        if not self.record_attention:
            raise RuntimeError("attention_maps() needs PwWSampler(..., record_attention=True)")
        m, (h, w) = self.m, self.latents.shape[-2:]
        total = torch.zeros((m, MAX_RECORDED_REGIONS, h, w), dtype=torch.float32, device=self.device)
        for _, hr, wr, acc in self._rec_levels:
            mean = acc.sum(1) / acc.shape[1]                                   # head mean: [m, N, 16]
            grid = mean.view(m, hr, wr, MAX_RECORDED_REGIONS).permute(0, 3, 1, 2)
            total += F.interpolate(grid, size=(h, w), mode="bilinear", align_corners=False)
        total /= max(1, self._rec_calls * self._step_no)
        return [total[i, :r].cpu() for i, r in enumerate(self._region_counts)]

    def _set_up_control(self, nets, images, weights, guesses, starts, ends):
        """Validate every unit's arguments (per-unit lists); embed the ControlNets' hints, run every adapter once on
        its hints, stack the ControlNet scale tables and sum the adapter features of every active set, and build the
        ControlNets' context."""
        from .adapter import T2IAdapter, adapter_scales, align_features, unet_level_sizes
        from .controlnet import ControlNetModel
        unet, m, U = self.unet, self.m, len(nets)
        h, w = self.latents.shape[-2:]
        params = inspect.signature(unet.forward).parameters
        ucfg = getattr(unet, "config", None)
        is_adapter = [isinstance(net, T2IAdapter) for net in nets]
        for u, (net, start, end) in enumerate(zip(nets, starts, ends)):
            def arg(name):           # the argument, with the unit's index when there are several
                return f"{name}[{u}]" if U > 1 else name
            if is_adapter[u]:
                if "down_intrablock_additional_residuals" not in params:
                    raise TypeError(f"the UNet ({type(unet).__name__}) does not take "
                                    "down_intrablock_additional_residuals, so it cannot take a T2I-Adapter")
                uch = getattr(ucfg, "block_out_channels", None)
                if uch is None or tuple(uch) != tuple(net.channels):
                    raise ValueError(f"{arg('controlnet')}: a T2I-Adapter of channels {list(net.channels)} does not "
                                     f"match the UNet's block_out_channels {None if uch is None else list(uch)}")
            elif not isinstance(net, ControlNetModel):
                raise TypeError(f"{arg('controlnet')} must be a paint_with_words_sd_b200.controlnet.ControlNetModel or "
                                f"a paint_with_words_sd_b200.adapter.T2IAdapter, got {type(net).__name__}")
            else:
                if "down_block_additional_residuals" not in params or "mid_block_additional_residual" not in params:
                    raise TypeError(f"the UNet ({type(unet).__name__}) does not take down_block_additional_residuals "
                                    "/ mid_block_additional_residual, so it cannot take a controlnet")
                ccfg = net.config
                for name in ("block_out_channels", "layers_per_block", "cross_attention_dim"):
                    if getattr(ucfg, name, None) != getattr(ccfg, name):
                        raise ValueError(f"{arg('controlnet')} config {name} = {getattr(ccfg, name)} does not match "
                                         f"the UNet's {getattr(ucfg, name, None)}")
                if ccfg.in_channels != 4:
                    raise ValueError(f"{arg('controlnet')} config in_channels = {ccfg.in_channels}: a ControlNet takes "
                                     "the 4 latent channels")
            if not start <= end:
                raise ValueError(f"{arg('control_guidance_start')} ({start}) must not exceed "
                                 f"{arg('control_guidance_end')} ({end})")
            if images[u] is None:
                raise ValueError(f"controlnet needs a {arg('control_image')} (one [1, 3, H, W] tensor per image)")
            images[u] = _per_image(images[u], m, arg("control_image"), torch.is_tensor)
            for i, img in enumerate(images[u]):
                if tuple(img.shape) != (1, 3, 8 * h, 8 * w):
                    raise ValueError(f"{arg('control_image')} {i} is {tuple(img.shape)}; expected (1, 3, {8 * h}, "
                                     f"{8 * w}): 8x the latent size {h}x{w}")
            weights[u] = _per_image(weights[u], m, arg("controlnet_conditioning_scale"),
                                    lambda s: isinstance(s, (int, float)) and not isinstance(s, bool))
        # guess-mode routing is global (hook_pww.py:39-53, 199): if any unit is in guess mode, every unit's residuals
        # and features go to the cond half only, and every ControlNet runs on the m cond rows
        self._nets, self._is_adapter, self.guess_mode = list(nets), is_adapter, any(guesses)
        n = len(self.timesteps)
        self._active_sets = [tuple(control_step_active(i, n, s, e) for s, e in zip(starts, ends)) for i in range(n)]
        self._control_active = [any(a) for a in self._active_sets]
        dev, udtype = self.device, _module_dtype(unet)
        rows = m if self.guess_mode else 2 * m
        sizes = unet_level_sizes(h, w)
        self._hints, feats = [], {}         # per unit: a ControlNet's embedded hints (None for an adapter); features
        for u, (net, imgs) in enumerate(zip(nets, images)):
            with torch.no_grad():                                                       # once: step-invariant
                hint = torch.cat([img.to(dev) for img in imgs], 0)
                if is_adapter[u]:
                    # PlugableAdapter.forward runs once and caches; the features go to the UNet's type
                    out = [f.to(udtype) for f in align_features(net(hint), sizes)]
                else:
                    out = [net.embed_condition(hint)]
            if not self.guess_mode:
                out = [torch.cat([t, t], 0) for t in out]                              # rows i and m + i share image i
            out = [t.contiguous(memory_format=torch.channels_last) if t.is_cuda else t for t in out]
            if is_adapter[u]:
                feats[u] = out
            self._hints.append(None if is_adapter[u] else out[0])
        tables = [(adapter_scales(wt, g) if ad else control_scales(wt, g, len(net.controlnet_down_blocks) + 1))[:, :rows]
                  for net, wt, g, ad in zip(nets, weights, guesses, is_adapter)]
        # per active set A that occurs, the active ControlNets' tables stacked: [|A|, levels, rows].  One unit's table is
        # the UNet inject's CONTROL_SCALES; two or more are applied in the combine, and the UNet adds the sum at scale 1
        self._combine_scales = {}
        # ... and the active adapters' scaled features summed level by level in unit order (hook_pww.py:136-139), once
        # here: 4 tensors at fixed addresses that the set's steps (and captured graphs) hand to the UNet
        self._adapter_sums = {}
        for a in set(self._active_sets):
            cn = [u for u in range(U) if a[u] and not is_adapter[u]]
            if cn:
                self._combine_scales[a] = torch.stack([tables[u] for u in cn], 0).contiguous().to(dev)
            ad = [u for u in range(U) if a[u] and is_adapter[u]]
            if ad:
                per_unit = [feats[u] for u in ad]
                scales = torch.stack([tables[u] for u in ad], 0).contiguous().to(dev)
                with torch.no_grad():
                    if fused_ops.is_fast(per_unit[0][0]):
                        self._adapter_sums[a] = fused_ops.control_combine(
                            per_unit, scales, [torch.empty_like(f) for f in per_unit[0]])
                    else:
                        self._adapter_sums[a] = combine_control_residuals(per_unit, scales)
        # the ControlNets' own dict: the plain text context (cond rows only in guess mode), no weight maps, so every
        # cross-attention call is unbiased; its K/V are staged once like the UNet's (the cache is keyed by module, so
        # the units share the dict, and a model that appears twice its K/V)
        text = self._ctx["CONTEXT_TENSOR"]
        self._control_ctx = {"CONTEXT_TENSOR": text[:m] if self.guess_mode else text,
                             "CROSS_ATTENTION_WEIGHT_ORIG": 0, "WEIGHT_FUNCTION": _zero_weight_function,
                             "SIGMA": 0.0, "KV_CACHE": {}}

    def step_forms(self) -> List[tuple]:
        """float64 (alpha, a, b, [beta0..beta3], gamma) of every step of this run (`scheduler.step_form`); the run's
        first step has no history."""
        sch = self.scheduler
        return [step_form(sch, sch.step_index_of(t), first=(i == 0)) for i, t in enumerate(self.timesteps)]

    def _build_rows(self) -> torch.Tensor:
        """[steps, _G + 2m + 6] fp32: every step's row.  The step form ends with the history slot this step writes and
        the noise row it reads."""
        sch, zeros = self.scheduler, [0.0] * self.m
        rows = []
        for i, (t, (alpha, a, b, beta, gamma)) in enumerate(zip(self.timesteps, self.step_forms())):
            si = sch.step_index_of(t)
            sigma = float(sch.sigmas[si])
            gs = [g_of_sigma(f, pr, sch.sigmas[si]) for f, pr in zip(self._fns, self._probed)]
            rows.append([sigma, 1.0 / math.sqrt(sigma * sigma + 1.0), float(t), *beta, *gs, *zeros,
                         alpha, a, b, gamma, float(i % self._hist_len), float(i)])
        return torch.tensor(rows, dtype=torch.float32)

    def _merge_contexts(self, conds, unconds) -> dict:
        """Batch the per-image dicts: CONTEXT_TENSOR -> [2m,T,Dc]; weight maps -> [m,N,T] stacks;
        WMAP_INDEX = [0..m-1, -1 x m] with -1 also for images whose weight function is zero; STAT_KIND = the probed
        statistic of every image (uncond images: max, ignored)."""
        m = self.m
        lengths = {int(c["CONTEXT_TENSOR"].shape[1]) for c in list(conds) + list(unconds)}
        if len(lengths) != 1:
            raise ValueError(f"all images of a sampler need the same text length (got T = {sorted(lengths)}); encode them "
                             "with the same max_prompt_chunks or use one sampler per length")
        ctx = {"CONTEXT_TENSOR": torch.cat([c["CONTEXT_TENSOR"] for c in conds] +
                                           [u["CONTEXT_TENSOR"] for u in unconds], 0).to(self.device)}
        for key in conds[0]:
            if not key.startswith("CROSS_ATTENTION_WEIGHT_"):
                continue
            vals = [c[key] for c in conds]
            if key == "CROSS_ATTENTION_WEIGHT_ORIG":
                ctx[key] = vals[0] if m == 1 else 0   # ORIG fallback is a single-image path ...
                if m > 1 and any(isinstance(v, torch.Tensor) for v in vals):
                    ctx["ORIG_FALLBACK_DROPPED"] = True   # ... and a level that would need it raises instead of losing its bias
                continue
            if all(isinstance(v, torch.Tensor) for v in vals):
                dense = torch.stack([v.detach().to("cpu", torch.float32) for v in vals], 0).contiguous()
                ctx[key] = dense.to(self.device)
                packed = pack_weight_map(dense)      # host-side set-up, like the map builder itself
                if packed is not None:
                    n = int(key.rsplit("_", 1)[1])
                    ctx[packed_key(n)] = (packed[0].to(self.device), packed[1].to(self.device))
            else:
                ctx[key] = 0
        ctx["WMAP_INDEX"] = torch.tensor([-1 if pr.is_zero else i for i, pr in enumerate(self._probed)] + [-1] * m,
                                         dtype=torch.int32, device=self.device)
        ctx["STAT_KIND"] = torch.tensor([STAT_MAX if pr.is_zero else pr.stat for pr in self._probed] + [STAT_MAX] * m,
                                        dtype=torch.int32, device=self.device)
        ctx["WEIGHT_FUNCTION"] = self.weight_function
        ctx["SIGMA"] = None
        ctx["KV_CACHE"] = {}       # to_k/to_v of the text context are step-invariant: computed at the first step
        # scratch of the attention launches, owned by this sampler: its captured graphs never see a buffer that another
        # sampler or a later, larger call replaced
        ctx["PWW_SCRATCH"] = (torch.zeros(max(64, 2 * m), dtype=torch.float32, device=self.device),
                              torch.zeros(_native.lib().pww_xattn_fused_workspace_bytes(), dtype=torch.uint8,
                                          device=self.device))
        return ctx

    # -- one step, expressed only with device tensors / device scalars --------------------------
    def _step_body(self, active: tuple = ()):
        m, (h, w) = self.m, self.latents.shape[-2:]
        L = _native.lib()
        stream = torch.cuda.current_stream(self.device).cuda_stream
        p = self._params
        # the UNet input in the UNet's own dtype (the reference runs under autocast): [2m, C, h, w], rows i and m + i
        # both fp16(latents_i / sqrt(sigma^2 + 1)) [+ the inpaint channels]
        _native.check(L.pww_sampler_input(self.latents.data_ptr(), p[_SCALE:].data_ptr(),
                                          None if self.extra_input is None else self.extra_input.data_ptr(),
                                          self._unet_in.data_ptr(), _dtype_code(self._unet_in.dtype), m,
                                          self._unet_in.shape[1], h, w, stream), "pww_sampler_input")
        t = p[_T:_T + 1]
        residuals = {}
        if active in self._combine_scales:
            # each active ControlNet sees the 4 latent channels of the UNet input (hook_pww.py:113-119), only the cond
            # rows in guess mode (the uncond rows' residuals would be discarded)
            x = self._unet_in[:m, :4] if self.guess_mode else self._unet_in[:, :4]
            outs = [net(x, t, encoder_hidden_states=self._control_ctx, controlnet_cond_embedding=hint,
                        return_dict=False)
                    for net, hint, on, ad in zip(self._nets, self._hints, active, self._is_adapter) if on and not ad]
            per_unit = [list(d) + [md] for d, md in outs]
            scales = self._combine_scales[active]
            if len(scales) == 1:
                # one active unit: the UNet's inject scales its residuals (a captured graph keeps the table's address)
                *down, mid = per_unit[0]
                self._ctx["CONTROL_SCALES"] = scales[0]
            else:
                # several: their scaled residuals summed level by level in unit order (hook_pww.py:136-139), in place
                # into the first active unit's, then added by the UNet at scale 1
                self._ctx.pop("CONTROL_SCALES", None)
                if fused_ops.is_fast(per_unit[0][0]):
                    *down, mid = fused_ops.control_combine(per_unit, scales)
                else:
                    *down, mid = combine_control_residuals(per_unit, scales)
            residuals = {"down_block_additional_residuals": down, "mid_block_additional_residual": mid}
        if active in self._adapter_sums:
            # the active adapters' summed features, added inside the encoder levels' last residual epilogues
            residuals["down_intrablock_additional_residuals"] = self._adapter_sums[active]
        eps = self.unet(self._unet_in, t, encoder_hidden_states=self._ctx, **residuals).sample
        if tuple(eps.shape) != (2 * m, 4, h, w) or eps.device != self.device:
            raise ValueError(f"the UNet returned {tuple(eps.shape)} on {eps.device}; expected {(2 * m, 4, h, w)}")
        # CFG with the per-image scale, then the step form; eps is read in place through its strides
        _native.check(L.pww_sampler_update(eps.data_ptr(), _dtype_code(eps.dtype), *eps.stride(),
                                           self.latents.data_ptr(), self._derivs.data_ptr(), self._hist_len,
                                           None if self._noise is None else self._noise.data_ptr(),
                                           self._gscale.data_ptr(), p[_BETA:].data_ptr(), p[self._form:].data_ptr(),
                                           m, h, w, stream), "pww_sampler_update")
        _native.launch_count += 2

    def _set_step_scalars(self, i: int, step_index: int):
        self._params.copy_(self._rows[i])
        self._ctx["SIGMA"] = self.scheduler.sigmas[step_index]

    # -- host-buffer interface (what bench.py's e2e leg drives) -----------------------------------
    def device_inputs(self) -> Dict[str, torch.Tensor]:
        """Persistent device tensors a step reads: latents, the text context and the stacked weight maps.
        Copying new values INTO them (same addresses) is valid between graph replays."""
        d = {"latents": self.latents, "CONTEXT_TENSOR": self._ctx["CONTEXT_TENSOR"]}
        for k, v in self._ctx.items():
            if k.startswith("CROSS_ATTENTION_PACKED_"):
                d[k + "_M"], d[k + "_C"] = v                       # packed map + token column index
            elif k.startswith("CROSS_ATTENTION_WEIGHT_") and isinstance(v, torch.Tensor) and v.is_cuda:
                n = k.rsplit("_", 1)[1]
                if n.isdigit() and packed_key(int(n)) not in self._ctx:
                    d[k] = v                                       # dense map (only when it could not be packed)
        return d

    def stage_from_host(self, pinned: Dict[str, torch.Tensor]) -> int:
        """Async H2D copy of this step's inputs from pinned host buffers; returns bytes copied."""
        dev = self.device_inputs()
        n = 0
        for k, h in pinned.items():
            dev[k].copy_(h, non_blocking=True)
            n += h.numel() * h.element_size()
        if "CONTEXT_TENSOR" in pinned and self._ctx.get("KV_CACHE"):
            # the cached K/V follow the new context: 16 small GEMMs, replayed as one CUDA graph (the ControlNet's
            # context is a view of the same tensor, so its cached K/V are refreshed too)
            ctxs = [self._ctx] + ([self._control_ctx] if self._combine_scales else [])

            def refresh():
                for c in ctxs:
                    _attention.refresh_kv_cache(c)
            if not self.use_graph:
                refresh()
            else:
                if self._kv_graph is None:
                    self._kv_graph, _ = self._capture(refresh, warmup=1)
                self._kv_graph.replay()
        return n

    def restart(self, latents: Optional[torch.Tensor] = None):
        """Rewind to step 0 (empty history, the first noise row), optionally with new latents."""
        self._step_no = 0
        self._derivs.zero_()
        for *_, acc in self._rec_levels:
            acc.zero_()
        if latents is not None:
            self.latents.copy_(latents)

    def step(self):
        if not self.latents.is_cuda:
            raise RuntimeError("PwWSampler steps run on a CUDA device (the sampler kernels have no CPU version)")
        i = self._step_no
        step_index = self.scheduler.step_index_of(self.timesteps[i])
        self._set_step_scalars(i, step_index)
        active = self._active_sets[i]
        if not self.use_graph:
            self._step_body(active)
        else:
            # one graph per set of active ControlNets (at most 2U + 1 over a run), each captured at the first step
            # that needs it; its two warm-up steps are undone, so the replay below is this step
            if active not in self._graphs:
                snap = [self.latents.clone(), self._derivs.clone()] + [acc.clone() for *_, acc in self._rec_levels]
                self._graphs[active] = self._capture(lambda: self._step_body(active), warmup=2)
                for buf, old in zip([self.latents, self._derivs] + [acc for *_, acc in self._rec_levels], snap):
                    buf.copy_(old)
            self._graphs[active][0].replay()
        self._step_no += 1

    def _capture(self, fn: Callable[[], None], warmup: int) -> Tuple["torch.cuda.CUDAGraph", int]:
        """`fn` captured in a CUDA graph after `warmup` eager runs on a side stream (allocator, cuDNN / cuBLAS
        autotuning); returns the graph and the native launches it holds."""
        s = torch.cuda.Stream(device=self.device)
        s.wait_stream(torch.cuda.current_stream(self.device))
        with torch.cuda.stream(s):
            for _ in range(warmup):
                fn()
        torch.cuda.current_stream(self.device).wait_stream(s)
        g = torch.cuda.CUDAGraph()
        before = _native.launch_count
        with torch.cuda.graph(g):
            fn()
        return g, _native.launch_count - before

    @property
    def native_launches_per_step(self) -> Optional[int]:
        """Native launches of the captured step (the step with every ControlNet, if there are any); None until
        captured."""
        return self._graphs.get((True,) * len(self._nets), (None, None))[1]

    @property
    def native_launches_per_step_without_control(self) -> Optional[int]:
        """Native launches of a ControlNet's captured step outside its window; None until captured or without one."""
        return self._graphs.get((False,) * len(self._nets), (None, None))[1] if self._nets else None

    @property
    def native_launches_per_active_set(self) -> Dict[tuple, int]:
        """Native launches of every captured step, keyed by its active set: one bool per ControlNet unit (() without
        a ControlNet)."""
        return {a: launches for a, (_, launches) in self._graphs.items()}

    def run(self, num_steps: Optional[int] = None) -> torch.Tensor:
        n = len(self.timesteps) - self._step_no if num_steps is None else num_steps
        with torch.no_grad():
            for _ in range(n):
                self.step()
        return self.latents


@torch.no_grad()
def paint_with_words(
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
    init_image: Optional[Image.Image] = None,
    strength: float = 0.5,
    return_latents: bool = False,
    max_prompt_chunks: int = 1,
    torch_dtype: Optional[torch.dtype] = None,
    controlnet=None,
    control_image: Union[None, Image.Image, Sequence[Image.Image]] = None,
    controlnet_conditioning_scale: Union[float, Sequence] = 1.0,
    guess_mode: Union[bool, Sequence[bool]] = False,
    control_guidance_start: Union[float, Sequence[float]] = 0.0,
    control_guidance_end: Union[float, Sequence[float]] = 1.0,
    return_attention_maps: bool = False,
):
    """paint_with_words.py:391-510.  Returns one PIL.Image (or the final latents with return_latents).
    `max_prompt_chunks` (1 .. 3): a prompt longer than 75 tokens fills up to that many 77-token CLIP chunks instead of
    being truncated (conditioning.chunk_prompt); 1 is the reference's behaviour.
    `torch_dtype` is passed to `pww_load_tools` when this call loads the models (torch.bfloat16 for a bf16 UNet); with
    `preloaded_utils` the UNet's own dtype decides.
    ControlNet (the reference's PwW + ControlNet extension): `controlnet` from `pww_load_controlnet`, `control_image`
    a PIL image of the colour map's size (scribble, edges, pose, ...) that fixes the layout while the colour map says
    which words go where; `controlnet_conditioning_scale`, `guess_mode` and the guidance window as in `PwWSampler`.
    Several ControlNets (e.g. pose for the figure, edges for the background): `controlnet` a list of up to 10,
    `control_image` a list with one such image per ControlNet, and the other four arguments one value or one per
    ControlNet.  A T2I-Adapter from `pww_load_adapter` is a unit too, alone or in the list, with the same arguments.
    `return_attention_maps=True` returns (image, RegionAttention): the per-region cross-attention maps of the cond image
    recorded inside the attention kernels over the whole run, with each region's adherence to its painted area."""
    control = _control_arguments(controlnet, control_image, color_map_image.size, "color_map_image",
                                 controlnet_conditioning_scale, guess_mode, control_guidance_start,
                                 control_guidance_end)
    tools = _tools(preloaded_utils, device, scheduler_type, local_model_path, hf_model_path, model_token, torch_dtype)
    vae, unet, text_encoder, tokenizer, scheduler = tools
    scheduler.set_timesteps(num_inference_steps)
    if init_image is None:
        cond, uncond, latents = _txt2img_inputs(tools, device, color_map_image, color_context, input_prompt,
                                                unconditional_input_prompt, seed, max_prompt_chunks)
        timesteps = scheduler.timesteps
    else:
        _, _, cond, uncond = _encode_text_color_inputs(
            text_encoder, tokenizer, device, color_map_image, color_context, input_prompt, unconditional_input_prompt,
            max_prompt_chunks=max_prompt_chunks)
        # the reference draws img2img's noise from the global RNG as it stands: unseeded here
        latents, timesteps = _img2img_latents(vae, scheduler, init_image, num_inference_steps, strength, device)
    sampler = PwWSampler(unet, scheduler, [cond], [uncond], latents, weight_function, guidance_scale,
                         timesteps=timesteps, noise_seed=seed, record_attention=return_attention_maps, **control)
    result = _result(vae, sampler.run(), return_latents)
    if not return_attention_maps:
        return result
    return result, _region_attention(sampler.attention_maps()[0], cond, color_context, color_map_image)


def _tools(preloaded_utils, device, scheduler_type, local_model_path, hf_model_path, model_token, torch_dtype):
    """The caller's (vae, unet, text_encoder, tokenizer, scheduler), or `pww_load_tools`'s when it passes none."""
    if preloaded_utils is not None:
        return preloaded_utils
    return pww_load_tools(device, scheduler_type, local_model_path=local_model_path, hf_model_path=hf_model_path,
                          model_token=model_token, torch_dtype=torch_dtype)


def _txt2img_inputs(tools, device, color_map_image, color_context, input_prompt, unconditional_input_prompt, seed,
                    max_prompt_chunks) -> Tuple[dict, dict, torch.Tensor]:
    """One txt2img image's (cond, uncond, latents): its text and colour contexts, and its seeded initial noise scaled
    by the scheduler's initial sigma (so `scheduler.set_timesteps` comes first)."""
    _, unet, text_encoder, tokenizer, scheduler = tools
    width, height = color_map_image.size
    extra_seeds, seperated_word_contexts, cond, uncond = _encode_text_color_inputs(
        text_encoder, tokenizer, device, color_map_image, color_context, input_prompt, unconditional_input_prompt,
        max_prompt_chunks=max_prompt_chunks)
    latents = initial_latents((1, unet.in_channels, height // 8, width // 8), seed, extra_seeds,
                              seperated_word_contexts).to(device)
    return cond, uncond, latents * scheduler.init_noise_sigma


def _img2img_latents(vae, scheduler, init_image, num_inference_steps: int, strength: float, device,
                     generator: Optional[torch.Generator] = None) -> Tuple[torch.Tensor, torch.Tensor]:
    """(latents, timesteps) of an img2img run: the last `strength` of the schedule, and the init image's VAE latents
    noised to its first timestep with noise from `generator` (None: the global RNG)."""
    init_timestep = min(int(num_inference_steps * strength), num_inference_steps)
    t_start = max(num_inference_steps - init_timestep, 0)
    timesteps = scheduler.timesteps[t_start:]
    image = preprocess(init_image).to(device=device)
    init_latents = 0.18215 * vae.encode(image.to(_module_dtype(vae, image.dtype))).latent_dist.sample().float()
    noise = torch.randn(init_latents.shape, generator=generator).to(device)
    return scheduler.add_noise(init_latents, noise, timesteps[:1]), timesteps


def _result(vae, latents: torch.Tensor, return_latents: bool):
    """What the public functions return for one image: its final latents, or the PIL image they decode to."""
    return latents if return_latents else _pil_from_latents(vae, latents)[0]


@dataclasses.dataclass
class RegionAttention:
    """Where each painted word looked, from `return_attention_maps=True`.
    labels    : the `color_context` labels, in order (region r = entry r)
    maps      : fp32 [R, h, w] at latent resolution: mean softmax mass region r's tokens receive (PwWSampler.attention_maps)
    coverage  : fp32 [R, h, w]: the fraction of each latent pixel that region r's colour covers in the colour map
    adherence : fp32 [R]: sum(maps * coverage) / sum(maps) per region -- the share of the region's attention that falls
                inside its painted area (NaN for a region whose label is not in the prompt)"""
    labels: List[str]
    maps: torch.Tensor
    coverage: torch.Tensor
    adherence: torch.Tensor


def region_adherence(maps: torch.Tensor, coverage: torch.Tensor, has_tokens: Sequence[bool]) -> torch.Tensor:
    """fp32 [R]: sum(maps[r] * coverage[r]) / sum(maps[r]) for every region with tokens, NaN for the others."""
    num = (maps * coverage).flatten(1).sum(1)
    den = maps.flatten(1).sum(1)
    out = num / den
    out[~torch.tensor([bool(t) for t in has_tokens], dtype=torch.bool)] = float("nan")
    return out.to(torch.float32)


def region_coverage(color_map_image: Image.Image, color_context: dict, size: Tuple[int, int]) -> torch.Tensor:
    """fp32 [R, h, w]: region r's binary colour mask (exact colour match, as the conditioning builder matches it)
    area-averaged to the latent size (h, w)."""
    pixels = np.array(color_map_image.convert("RGB"))
    masks = [torch.from_numpy((pixels == _rgb_of(c)).all(axis=-1)).to(torch.float32) for c in color_context]
    if not masks:
        return torch.zeros((0,) + tuple(size), dtype=torch.float32)
    return F.interpolate(torch.stack(masks, 0)[:, None], size=tuple(size), mode="area")[:, 0]


def _region_attention(maps: torch.Tensor, cond: dict, color_context: dict, color_map_image) -> RegionAttention:
    """The RegionAttention of one image from its recorded maps, cond dict and colour inputs."""
    labels = [spec.rpartition(",")[0]
              for spec in _extract_seed_and_sigma_from_context(dict(color_context))[0].values()]
    coverage = region_coverage(color_map_image, color_context, tuple(maps.shape[-2:]))
    ridx = cond[REGION_INDEX_KEY]
    has_tokens = [bool((ridx == r).any()) for r in range(len(labels))]
    maps = maps[:len(labels)]
    return RegionAttention(labels, maps, coverage, region_adherence(maps, coverage, has_tokens))


def _control_arguments(controlnet, control_image, size: Tuple[int, int], size_of: str, conditioning_scale,
                       guess_mode: bool, start: float, end: float) -> dict:
    """PwWSampler's ControlNet keyword arguments from the public ones, as per-unit lists (`_control_units`), {} without
    a controlnet.  Every hint image must be `size` (W, H); with a list of ControlNets, `control_image` is a list of one
    such image per unit."""
    if controlnet is None:
        if control_image is not None:
            raise ValueError("control_image is given but controlnet is None")
        return {}
    nets, images, weights, guesses, starts, ends = _control_units(controlnet, control_image, conditioning_scale,
                                                                  guess_mode, start, end)
    indexed = isinstance(controlnet, (list, tuple))       # a list's images are named by unit
    for u, image in enumerate(images):
        name = f"control_image[{u}]" if indexed else "control_image"
        if not isinstance(image, Image.Image):
            raise ValueError(f"controlnet needs a {name} (a PIL image of the {size_of} size {size}), got "
                             f"{type(image).__name__}")
        if image.size != tuple(size):
            raise ValueError(f"{name} is {image.size}; it must have the {size_of} size {tuple(size)}")
    return dict(controlnet=nets, control_image=[control_image_tensor(image) for image in images],
                controlnet_conditioning_scale=weights, guess_mode=guesses, control_guidance_start=starts,
                control_guidance_end=ends)


# the per-image keyword arguments of paint_with_words that paint_with_words_batch takes per entry
BATCH_SETTING_KEYS = ("color_context", "color_map_image", "input_prompt", "unconditional_input_prompt", "seed",
                      "weight_function", "guidance_scale", "max_prompt_chunks", "control_image",
                      "controlnet_conditioning_scale")


def _batch_settings(settings) -> List[dict]:
    """Every entry with paint_with_words's defaults filled in; unknown keys and img2img raise ValueError."""
    params = inspect.signature(paint_with_words).parameters
    out = []
    for i, entry in enumerate(settings):
        unknown = set(entry) - set(BATCH_SETTING_KEYS)
        if unknown & {"init_image", "strength"}:
            raise ValueError(f"settings[{i}]: init_image / strength cannot be batched (img2img draws its noise from the "
                             "global RNG); call paint_with_words for that image")
        if unknown:
            raise ValueError(f"settings[{i}]: unknown keys {sorted(unknown)}; the per-image keys are "
                             f"{', '.join(BATCH_SETTING_KEYS)}")
        full = {k: params[k].default for k in BATCH_SETTING_KEYS}
        full.update(entry)
        if full["color_map_image"] is None:
            raise ValueError(f"settings[{i}]: color_map_image is required")
        out.append(full)
    return out


def batch_groups(keys: Sequence, max_batch_size: int) -> List[List[int]]:
    """Indices of the entries grouped by key (groups in order of first appearance, input order inside a group), each
    group cut into runs of at most `max_batch_size` (>= 1: paint_with_words_batch checks it before it loads any
    model): one sampler per run.  A key of None is never shared."""
    groups: Dict[object, List[int]] = {}
    for i, key in enumerate(keys):
        groups.setdefault(("solo", i) if key is None else key, []).append(i)
    return [g[j:j + max_batch_size] for g in groups.values() for j in range(0, len(g), max_batch_size)]


@torch.no_grad()
def paint_with_words_batch(
    settings: Sequence[dict],
    num_inference_steps: int = 30,
    scheduler_type=LMSDiscreteScheduler,
    device: str = "cuda:0",
    local_model_path: Optional[str] = None,
    hf_model_path: Optional[str] = "synthetic:sd15",
    preloaded_utils: Optional[Tuple] = None,
    model_token: Optional[str] = None,
    max_batch_size: int = 8,
    return_latents: bool = False,
    torch_dtype: Optional[torch.dtype] = None,
    controlnet=None,
    guess_mode: Union[bool, Sequence[bool]] = False,
    control_guidance_start: Union[float, Sequence[float]] = 0.0,
    control_guidance_end: Union[float, Sequence[float]] = 1.0,
    return_attention_maps: bool = False,
):
    """Many images, each with its own settings, in as few samplers as possible.  `settings[i]` is a dict of the
    per-image keyword arguments of `paint_with_words` (BATCH_SETTING_KEYS: color_context, color_map_image, input_prompt,
    unconditional_input_prompt, seed, weight_function, guidance_scale, max_prompt_chunks, control_image,
    controlnet_conditioning_scale); missing keys take paint_with_words's defaults.  Returns a list of PIL images (or
    [1,4,h,w] latents) in input order; image i equals `paint_with_words(**settings[i])` up to fp16 noise.
    With `controlnet` (one for the batch, with `guess_mode` and the guidance window) every entry needs a
    `control_image` of its colour map's size; its `controlnet_conditioning_scale` is its own.  With a list of
    ControlNets (`guess_mode` and the window each one value or one per ControlNet), an entry's `control_image` is a list
    of one image per ControlNet and its `controlnet_conditioning_scale` one float or one per ControlNet.

    Entries of the same latent size and text length run in one `PwWSampler` of at most `max_batch_size` images (a
    2 * max_batch_size UNet batch with CFG), whatever their weight functions and guidance scales.  The default of 8 gave
    the most images/s of k = 1, 2, 4, 8 at 512x512 (BASELINE.md section 4) and bounds memory.  Sizes that are not multiples of 64 need the single-image weight-map fallback and
    run one image per sampler.  img2img (init_image / strength) is not batched.  `torch_dtype` as in
    `paint_with_words`.  `return_attention_maps=True` returns a list of (image, RegionAttention) pairs in input order
    (see `paint_with_words`)."""
    entries = _batch_settings(settings)
    if max_batch_size < 1:
        raise ValueError("max_batch_size must be >= 1")
    controls = []
    for i, e in enumerate(entries):
        try:
            controls.append(_control_arguments(controlnet, e["control_image"], e["color_map_image"].size,
                                               "color_map_image", e["controlnet_conditioning_scale"], guess_mode,
                                               control_guidance_start, control_guidance_end))
        except ValueError as err:
            raise ValueError(f"settings[{i}]: {err}") from err
    tools = _tools(preloaded_utils, device, scheduler_type, local_model_path, hf_model_path, model_token, torch_dtype)
    vae, unet, _, _, scheduler = tools
    scheduler.set_timesteps(num_inference_steps)
    encoded, keys = [], []
    for e in entries:
        cond, uncond, latents = _txt2img_inputs(tools, device, e["color_map_image"], dict(e["color_context"]),
                                                e["input_prompt"], e["unconditional_input_prompt"], e["seed"],
                                                e["max_prompt_chunks"])
        encoded.append((cond, uncond, latents))
        width, height = e["color_map_image"].size
        solo = width % 64 != 0 or height % 64 != 0
        keys.append(None if solo else (height // 8, width // 8, int(cond["CONTEXT_TENSOR"].shape[1])))
    results: List[Optional[torch.Tensor]] = [None] * len(entries)
    attention: List[Optional[RegionAttention]] = [None] * len(entries)
    for idx in batch_groups(keys, max_batch_size):
        control = controls[idx[0]]
        if control:         # the batch's ControlNets and windows; per unit, each image's own hint and weight
            units = range(len(control["controlnet"]))
            control = dict(control, control_image=[[controls[i]["control_image"][u] for i in idx] for u in units],
                           controlnet_conditioning_scale=[[controls[i]["controlnet_conditioning_scale"][u] for i in idx]
                                                          for u in units])
        sampler = PwWSampler(unet, scheduler, [encoded[i][0] for i in idx], [encoded[i][1] for i in idx],
                             torch.cat([encoded[i][2] for i in idx], 0),
                             [entries[i]["weight_function"] for i in idx], [entries[i]["guidance_scale"] for i in idx],
                             timesteps=scheduler.timesteps, noise_seed=[entries[i]["seed"] for i in idx],
                             record_attention=return_attention_maps, **control)
        latents = sampler.run()
        maps = sampler.attention_maps() if return_attention_maps else None
        for j, i in enumerate(idx):
            results[i] = latents[j:j + 1].clone()
            if maps is not None:
                attention[i] = _region_attention(maps[j], encoded[i][0], entries[i]["color_context"],
                                                 entries[i]["color_map_image"])
        del sampler
    images = [_result(vae, lat, return_latents) for lat in results]
    return list(zip(images, attention)) if return_attention_maps else images


def prepare_mask_and_masked_image(image, mask):
    """paint_with_words_inpaint.py:20-106 (PIL / ndarray inputs): mask binarised at 0.5, image in [-1,1],
    masked_image = image * (mask < 0.5)."""
    if isinstance(image, torch.Tensor) or isinstance(mask, torch.Tensor):
        if not (isinstance(image, torch.Tensor) and isinstance(mask, torch.Tensor)):
            raise TypeError("`image` and `mask` must both be tensors or both be PIL/ndarray")
        if image.ndim == 3:
            image = image.unsqueeze(0)
        if mask.ndim == 2:
            mask = mask[None, None]
        elif mask.ndim == 3:
            mask = mask.unsqueeze(0) if mask.shape[0] == 1 else mask.unsqueeze(1)
        if image.min() < -1 or image.max() > 1:
            raise ValueError("Image should be in [-1, 1] range")
        if mask.min() < 0 or mask.max() > 1:
            raise ValueError("Mask should be in [0, 1] range")
        mask = (mask >= 0.5).to(torch.float32)
        image = image.to(torch.float32)
    else:
        if isinstance(image, Image.Image):
            image = np.array(image.convert("RGB"))
        image = torch.from_numpy(image[None].transpose(0, 3, 1, 2)).to(torch.float32) / 127.5 - 1.0
        if isinstance(mask, Image.Image):
            mask = np.array(mask.convert("L")).astype(np.float32) / 255.0
        mask = torch.from_numpy((mask[None, None] >= 0.5).astype(np.float32))
    return mask, image * (mask < 0.5)


@torch.no_grad()
def paint_with_words_inpaint(
    color_context: Dict[Tuple[int, int, int], str] = {},
    color_map_image: Optional[Image.Image] = None,
    mask_image: Optional[Image.Image] = None,
    init_image: Image.Image = None,
    input_prompt: str = "",
    num_inference_steps: int = 150,
    guidance_scale: float = 7.5,
    seed: int = 0,
    scheduler_type=LMSDiscreteScheduler,
    device: str = "cuda:0",
    weight_function: Callable = default_weight_function,
    local_model_path: Optional[str] = None,
    hf_model_path: Optional[str] = "synthetic:sd15-inpaint",
    preloaded_utils: Optional[Tuple] = None,
    unconditional_input_prompt: str = "",
    model_token: Optional[str] = None,
    strength: float = 1.0,
    return_latents: bool = False,
    max_prompt_chunks: int = 1,
    torch_dtype: Optional[torch.dtype] = None,
    controlnet=None,
    control_image: Union[None, Image.Image, Sequence[Image.Image]] = None,
    controlnet_conditioning_scale: Union[float, Sequence] = 1.0,
    guess_mode: Union[bool, Sequence[bool]] = False,
    control_guidance_start: Union[float, Sequence[float]] = 0.0,
    control_guidance_end: Union[float, Sequence[float]] = 1.0,
    return_attention_maps: bool = False,
):
    """paint_with_words_inpaint.py:137-270: 9-channel UNet input cat[latents, mask, masked-image latents].
    `max_prompt_chunks`, `torch_dtype` and the ControlNet arguments as in `paint_with_words`; the colour map is resized
    to the init image, so `control_image` has the init image's size.  The ControlNet sees the 4 latent channels of
    the UNet input (hook_pww.py:113-119).  `return_attention_maps` as in `paint_with_words` (coverage from the resized
    colour map)."""
    width, height = init_image.size
    control = _control_arguments(controlnet, control_image, (width, height), "init_image (and resized color_map_image)",
                                 controlnet_conditioning_scale, guess_mode, control_guidance_start,
                                 control_guidance_end)
    vae, unet, text_encoder, tokenizer, scheduler = _tools(preloaded_utils, device, scheduler_type, local_model_path,
                                                           hf_model_path, model_token, torch_dtype)
    color_map_image = color_map_image.resize((width, height), Image.NEAREST)
    mask_image = mask_image.resize((width, height), Image.NEAREST)
    _, _, cond, uncond = _encode_text_color_inputs(
        text_encoder, tokenizer, device, color_map_image, color_context, input_prompt, unconditional_input_prompt,
        max_prompt_chunks=max_prompt_chunks)
    mask, masked_image = prepare_mask_and_masked_image(init_image, mask_image)

    scheduler.set_timesteps(num_inference_steps)
    # seeded before the VAE encode, which draws from the same (global) generator
    latents, timesteps = _img2img_latents(vae, scheduler, init_image, num_inference_steps, strength, device,
                                          generator=torch.manual_seed(seed))

    mask = F.interpolate(mask, size=(height // 8, width // 8)).to(device=device, dtype=latents.dtype)
    masked_image_latents = 0.18215 * vae.encode(masked_image.to(device=device, dtype=_module_dtype(vae, latents.dtype))).latent_dist.sample().float()
    mask = F.interpolate(mask, size=latents.shape[-2:], mode="nearest")
    masked_image_latents = F.interpolate(masked_image_latents, size=latents.shape[-2:], mode="nearest")
    total = latents.shape[1] + mask.shape[1] + masked_image_latents.shape[1]
    if total != unet.in_channels:
        raise ValueError(
            f"Incorrect configuration settings! The unet expects {unet.in_channels} input channels but received "
            f"num_channels_latents: {latents.shape[1]} + num_channels_mask: {mask.shape[1]} + "
            f"num_channels_masked_image: {masked_image_latents.shape[1]} = {total}.")
    sampler = PwWSampler(unet, scheduler, [cond], [uncond], latents, weight_function, guidance_scale,
                         extra_input=torch.cat([mask, masked_image_latents], 1).float(), timesteps=timesteps,
                         noise_seed=seed, record_attention=return_attention_maps, **control)
    result = _result(vae, sampler.run(), return_latents)
    if not return_attention_maps:
        return result
    return result, _region_attention(sampler.attention_maps()[0], cond, color_context, color_map_image)


# ---------------------------------------------------------------------------------------------
# pipeline classes (paint_with_words.py:513-842, paint_with_words_inpaint.py:273-575): API surface only
# ---------------------------------------------------------------------------------------------
class PipelineOutput:
    """Stand-in for diffusers' StableDiffusionPipelineOutput: `.images`, `.nsfw_content_detected`."""

    def __init__(self, images, nsfw_content_detected=False):
        self.images, self.nsfw_content_detected = images, nsfw_content_detected


class PaintWithWord_StableDiffusionPipeline:
    """Same constructor / `from_pretrained` / `plugin_cross_attention` / `__call__` surface as the reference class
    (paint_with_words.py:513-842); the work is `paint_with_words()` above (one `PwWSampler`).  Like the reference class
    it always uses its own LMS scheduler (paint_with_words.py:534-539) and has no regional blur (:574)."""

    def __init__(self, vae, text_encoder, tokenizer, unet, scheduler=None, safety_checker=None, feature_extractor=None,
                 requires_safety_checker: bool = False, controlnet=None):
        """`controlnet`: a `ControlNetModel` (`pww_load_controlnet`), or a list of them, that every call passing a
        `control_image` uses (with a list, `control_image` has one image per ControlNet)."""
        self.vae, self.text_encoder, self.tokenizer, self.unet = vae, text_encoder, tokenizer, unet
        self.safety_checker, self.feature_extractor = safety_checker, feature_extractor
        self.controlnet = controlnet
        self.scheduler = LMSDiscreteScheduler(beta_start=0.00085, beta_end=0.012, beta_schedule="scaled_linear",
                                              num_train_timesteps=1000)
        self.plugin_cross_attention()

    @classmethod
    def from_pretrained(cls, save_dir, device: str = "cuda:0", torch_dtype: Optional[torch.dtype] = None, **kwargs):
        """`torch_dtype` as in `pww_load_tools` (torch.bfloat16 for a bf16 UNet)."""
        vae, unet, text_encoder, tokenizer, scheduler = pww_load_tools(device, local_model_path=save_dir,
                                                                       torch_dtype=torch_dtype)
        return cls(vae=vae, text_encoder=text_encoder, tokenizer=tokenizer, unet=unet, scheduler=scheduler,
                   controlnet=kwargs.get("controlnet"))

    def plugin_cross_attention(self):
        """paint_with_words.py:556-559."""
        return _attention.patch_unet(self.unet)

    @property
    def device(self):
        return next(iter(self.unet.parameters())).device

    def _run(self, fn, prompt, color_map_image, color_context, weight_function, num_inference_steps, guidance_scale,
             negative_prompt, seed, output_type, return_dict, callback, callback_steps, **extra):
        if isinstance(prompt, (list, tuple)):
            if len(prompt) != 1:
                raise ValueError("the Paint-with-Words pipelines take one prompt per call (batch size 1, paint_with_words.py:445)")
            prompt = prompt[0]
        if isinstance(negative_prompt, (list, tuple)):
            negative_prompt = negative_prompt[0]
        tools = (self.vae, self.unet, self.text_encoder, self.tokenizer, self.scheduler)
        latents = fn(color_context=color_context, color_map_image=color_map_image, input_prompt=prompt,
                     num_inference_steps=num_inference_steps, guidance_scale=guidance_scale, seed=seed,
                     device=str(self.device), weight_function=weight_function, preloaded_utils=tools,
                     unconditional_input_prompt=negative_prompt or "", return_latents=True, **extra)
        if callback is not None:
            callback(num_inference_steps - 1, int(self.scheduler.timesteps[-1]), latents)
        if output_type == "latent":
            images = latents
        else:
            images = _pil_from_latents(self.vae, latents)
            if output_type != "pil":
                images = np.stack([np.asarray(im, dtype=np.float32) / 255.0 for im in images])
        return PipelineOutput(images, False) if return_dict else (images, False)

    @torch.no_grad()
    def __call__(self, prompt, color_map_image=None, color_context={}, weight_function: Callable = default_weight_function,
                 height=None, width=None, num_inference_steps: int = 30, guidance_scale: float = 7.5, negative_prompt="",
                 num_images_per_prompt: int = 1, eta: float = 0.5, seed: int = 0, generator=None, image=None, latents=None,
                 output_type: str = "pil", return_dict: bool = True, callback=None, callback_steps: int = 1,
                 max_prompt_chunks: int = 1, control_image=None, controlnet_conditioning_scale: float = 1.0,
                 guess_mode: bool = False, control_guidance_start: float = 0.0, control_guidance_end: float = 1.0):
        extra = {} if image is None else {"init_image": image, "strength": eta}
        extra["max_prompt_chunks"] = max_prompt_chunks
        extra.update(self._control(control_image, controlnet_conditioning_scale, guess_mode, control_guidance_start,
                                   control_guidance_end))
        return self._run(paint_with_words, prompt, color_map_image, dict(color_context), weight_function,
                         num_inference_steps, guidance_scale, negative_prompt, seed, output_type, return_dict, callback,
                         callback_steps, **extra)

    def _control(self, control_image, scale, guess_mode, start, end) -> dict:
        """The ControlNet keyword arguments of a call: none when it passes no control_image."""
        if control_image is None:
            return {}
        return dict(controlnet=self.controlnet, control_image=control_image, controlnet_conditioning_scale=scale,
                    guess_mode=guess_mode, control_guidance_start=start, control_guidance_end=end)


class PaintWithWord_StableDiffusionInpaintPipeline(PaintWithWord_StableDiffusionPipeline):
    """paint_with_words_inpaint.py:273-575: `__call__(prompt, image, mask_image, color_map_image, color_context, ...)`."""

    @torch.no_grad()
    def __call__(self, prompt, image=None, mask_image=None, color_map_image=None, color_context={},
                 weight_function: Callable = default_weight_function, height=None, width=None,
                 num_inference_steps: int = 30, guidance_scale: float = 7.5, negative_prompt="",
                 num_images_per_prompt: int = 1, eta: float = 1.0, seed: int = 0, generator=None, latents=None,
                 output_type: str = "pil", return_dict: bool = True, callback=None, callback_steps: int = 1,
                 max_prompt_chunks: int = 1, control_image=None, controlnet_conditioning_scale: float = 1.0,
                 guess_mode: bool = False, control_guidance_start: float = 0.0, control_guidance_end: float = 1.0):
        return self._run(paint_with_words_inpaint, prompt, color_map_image, dict(color_context), weight_function,
                         num_inference_steps, guidance_scale, negative_prompt, seed, output_type, return_dict, callback,
                         callback_steps, mask_image=mask_image, init_image=image, strength=eta,
                         max_prompt_chunks=max_prompt_chunks,
                         **self._control(control_image, controlnet_conditioning_scale, guess_mode,
                                         control_guidance_start, control_guidance_end))
