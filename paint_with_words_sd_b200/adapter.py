"""T2I-Adapter control units (the reference extension's `PlugableAdapter`, pww_controlnet/scripts/adapter.py).

An adapter is a small conv net that maps a hint image to one feature map per UNet encoder level.  It does not see the
latents or the timestep, so a sampler runs it once per hint and adds its (scaled) features inside the UNet's residual
epilogues at every controlled step (`UNet2DConditionModel.forward(down_intrablock_additional_residuals=...)`).

Two forms, with the reference's parameter names so a TencentARC v1 state dict loads with `strict=True`:

  * full (`Adapter(channels, nums_rb, cin, ksize, sk=True, use_conv=False)`: the sketch, image and keypose adapters):
    PixelUnshuffle(8), `conv_in` (3x3, cin -> C0), then `body.{i}` for i < 4 * nums_rb: ResNet blocks whose first
    block of each level after level 0 starts with a 2x2 average pool and `in_conv` (ksize, C_{l-1} -> C_l) where the
    width changes; a block is `block2(relu(block1(x))) + x` (the second `ResnetBlock` definition of adapter.py, the one
    Python binds).  A feature is taken after each level.
  * light (`Adapter_light(channels, nums_rb, cin)`: the color adapter): PixelUnshuffle(8), then per level `body.{i}`:
    [2x2 average pool for i > 0], `in_conv` (1x1, -> C_l / 4), nums_rb blocks `body.{i}.body.{j}` (3x3 convs),
    `out_conv` (1x1, -> C_l).

A hint is [R, 3, H, W] in [0, 1] (the ControlNet's hint format).  An adapter with cin == 64 takes its first channel
(adapter.py:101-104), one with cin == 192 all three.
"""
from __future__ import annotations

from typing import List, Optional, Sequence, Tuple

import torch
import torch.nn as nn
import torch.nn.functional as F

from .unet import UNetConfig

LEVELS = 4
# guess mode scales level l of an adapter unit by weight * ADAPTER_GUESS_SCALES[l].  hook_pww.py:130 writes this as
# `param.weight * [0.25, 0.62, 0.825, 1.0]`, a Python list product (a TypeError for a float weight, list repetition
# for an int); the per-level product is what it means, and what is computed here.
ADAPTER_GUESS_SCALES = (0.25, 0.62, 0.825, 1.0)
KINDS = ("full", "light")


class _Block(nn.Module):
    """A full adapter's ResNet block (sk=True, use_conv=False)."""

    def __init__(self, in_c: int, out_c: int, down: bool, ksize: int):
        super().__init__()
        ps = ksize // 2
        self.in_conv = nn.Conv2d(in_c, out_c, ksize, 1, ps) if in_c != out_c else None
        self.block1 = nn.Conv2d(out_c, out_c, 3, 1, 1)
        self.block2 = nn.Conv2d(out_c, out_c, ksize, 1, ps)
        self.down = down

    def forward(self, x):
        if self.down:
            x = F.avg_pool2d(x, 2, 2)
        if self.in_conv is not None:
            x = self.in_conv(x)
        return self.block2(F.relu(self.block1(x))) + x


class _LightBlock(nn.Module):
    def __init__(self, c: int):
        super().__init__()
        self.block1 = nn.Conv2d(c, c, 3, 1, 1)
        self.block2 = nn.Conv2d(c, c, 3, 1, 1)

    def forward(self, x):
        return self.block2(F.relu(self.block1(x))) + x


class _Extractor(nn.Module):
    """One level of the light adapter."""

    def __init__(self, in_c: int, inter_c: int, out_c: int, nums_rb: int, down: bool):
        super().__init__()
        self.in_conv = nn.Conv2d(in_c, inter_c, 1, 1, 0)
        self.body = nn.Sequential(*[_LightBlock(inter_c) for _ in range(nums_rb)])
        self.out_conv = nn.Conv2d(inter_c, out_c, 1, 1, 0)
        self.down = down

    def forward(self, x):
        if self.down:
            x = F.avg_pool2d(x, 2, 2)
        return self.out_conv(self.body(self.in_conv(x)))


class T2IAdapter(nn.Module):
    """A T2I-Adapter: `kind` "full" or "light", `channels` the UNet's block_out_channels (4 levels), `cin` 64 (one
    hint channel) or 192 (three), `nums_rb` blocks per level, `ksize` the full form's in_conv / block2 kernel size."""

    def __init__(self, kind: str, channels: Sequence[int], cin: int, nums_rb: int, ksize: int = 1):
        super().__init__()
        if kind not in KINDS:
            raise ValueError(f"adapter kind {kind!r}: one of {KINDS}")
        if cin not in (64, 192):
            raise ValueError(f"adapter cin = {cin}: 64 (one hint channel) or 192 (three)")
        if len(channels) != LEVELS or nums_rb < 1:
            raise ValueError(f"an adapter has {LEVELS} levels and nums_rb >= 1 (got {list(channels)}, {nums_rb})")
        self.kind, self.channels, self.cin, self.nums_rb, self.ksize = kind, tuple(channels), cin, nums_rb, ksize
        if kind == "full":
            self.conv_in = nn.Conv2d(cin, channels[0], 3, 1, 1)
            self.body = nn.ModuleList([
                _Block(channels[i - 1] if (i and not j) else channels[i], channels[i], bool(i and not j), ksize)
                for i in range(LEVELS) for j in range(nums_rb)])
        else:
            self.body = nn.ModuleList([_Extractor(cin if i == 0 else channels[i - 1], channels[i] // 4, channels[i],
                                                  nums_rb, i > 0) for i in range(LEVELS)])

    def forward(self, hint: torch.Tensor) -> List[torch.Tensor]:
        """[R, 3, H, W] hint images in [0, 1] (H, W multiples of 8) -> the 4 features [R, C_l, H / 8 / 2^l, W / 8 /
        2^l] (sizes rounded down at each pool), in the adapter's type, channels-last on CUDA."""
        if hint.dim() != 4 or hint.shape[1] != 3 or hint.shape[2] % 8 or hint.shape[3] % 8:
            raise ValueError(f"an adapter hint is [R, 3, H, W] with H and W multiples of 8, got {tuple(hint.shape)}")
        w = next(self.parameters())
        x = hint[:, :1] if self.cin == 64 else hint
        x = F.pixel_unshuffle(x.to(device=w.device, dtype=w.dtype), 8)
        if x.is_cuda:
            x = x.contiguous(memory_format=torch.channels_last)
        feats = []
        if self.kind == "full":
            x = self.conv_in(x)
            for i in range(LEVELS):
                for j in range(self.nums_rb):
                    x = self.body[i * self.nums_rb + j](x)
                feats.append(x)
        else:
            for blk in self.body:
                x = blk(x)
                feats.append(x)
        return feats


def adapter_scales(weights: Sequence[float], guess_mode: bool) -> torch.Tensor:
    """An adapter unit's scale table for m images: fp32 [4, rows].  Plain: rows = 2m, columns i and m + i hold
    weight_i at every level.  Guess mode: rows = m (only the cond half gets features), entry [l, i] = weight_i *
    ADAPTER_GUESS_SCALES[l]."""
    w = torch.tensor([float(s) for s in weights], dtype=torch.float64)
    if guess_mode:
        return (torch.tensor(ADAPTER_GUESS_SCALES, dtype=torch.float64)[:, None] * w[None, :]).to(torch.float32)
    return torch.cat([w, w]).to(torch.float32)[None, :].repeat(LEVELS, 1)


def unet_level_sizes(h: int, w: int, levels: int = LEVELS) -> List[Tuple[int, int]]:
    """(h_l, w_l) of the UNet's encoder levels at latent size h x w: its downsamplers are stride-2 3x3 convs with
    padding 1, which round up."""
    sizes = [(h, w)]
    for _ in range(levels - 1):
        h, w = (h + 1) // 2, (w + 1) // 2
        sizes.append((h, w))
    return sizes


def align_features(feats: Sequence[torch.Tensor], sizes: Sequence[Tuple[int, int]]) -> List[torch.Tensor]:
    """Each feature resized (nearest) to its level's size where they differ (hook_pww.py:55-59).  The adapter's
    average pools round down where the UNet's downsamplers round up, so an odd side at some level makes them
    differ."""
    out = []
    for f, (h, w) in zip(feats, sizes):
        if tuple(f.shape[-2:]) != (h, w):
            f = F.interpolate(f, size=(h, w), mode="nearest")
        out.append(f)
    return out


# the TencentARC v1 adapters: sketch / image / keypose are full with nums_rb=2, ksize=1; color is light with nums_rb=4
_SYNTHETIC_KINDS = {"full64": ("full", 64, 2), "full192": ("full", 192, 2), "light": ("light", 192, 4)}
_SYNTHETIC_CONFIGS = {"sd15": UNetConfig.sd15, "sd21": UNetConfig.sd21, "tiny": UNetConfig.tiny}


def build_adapter(cfg: UNetConfig, kind: str = "full", cin: int = 192, seed: int = 3, nums_rb: Optional[int] = None,
                  ksize: int = 1, dtype=torch.float32, device="cpu") -> T2IAdapter:
    """Seeded random weights (torch's default initialisation) for an adapter matching `cfg`'s block_out_channels,
    generated on the host (then cast / moved).  nums_rb defaults to the TencentARC v1 value of the kind (full 2, light
    4).  Every layer is random and nonzero, so the features are too, and a comparison of two paths that add them
    cannot pass by adding zeros.

    With torch's default initialisation alone, each conv shrinks its input's scale (by about sqrt(3) for a 1x1 conv),
    and the features of a scribble hint at 512x512 come out with a standard deviation of 0.04-0.14, where the SD1.5
    activations they are added to have 0.6-0.9: an adapter would barely move the result.  So a few layers get a fixed
    gain, weight and bias alike: the full form's conv_in x6 and its width-changing in_convs x sqrt(3), the light
    form's out_convs x4 (level 0) and x2.5 (levels 1-3).  That puts the features at a standard deviation of 0.7-0.86
    (full) and about 0.4 (light) at every level, for the sd15 and tiny configs, and finite in fp16."""
    nums_rb = (2 if kind == "full" else 4) if nums_rb is None else nums_rb
    with torch.random.fork_rng(devices=[]):
        torch.manual_seed(seed)
        net = T2IAdapter(kind, cfg.block_out_channels, cin, nums_rb, ksize)
    if kind == "full":
        gains = [(net.conv_in, 6.0)] + [(b.in_conv, 3.0 ** 0.5) for b in net.body if b.in_conv is not None]
    else:
        gains = [(e.out_conv, 4.0 if i == 0 else 2.5) for i, e in enumerate(net.body)]
    with torch.no_grad():
        for conv, k in gains:
            conv.weight.mul_(k)
            conv.bias.mul_(k)
    net.eval().requires_grad_(False)
    net = net.to(device=device, dtype=dtype)
    if torch.device(device).type == "cuda":
        net = net.to(memory_format=torch.channels_last)
    return net


def _infer(sd: dict) -> Tuple[str, Tuple[int, ...], int, int, int]:
    """(kind, channels, cin, nums_rb, ksize) of a state dict's keys and shapes; ValueError if it is not a full or
    light adapter of 4 levels."""
    def shape(key):
        t = sd.get(key)
        if not torch.is_tensor(t):
            raise ValueError(f"adapter state dict: {key} is missing")
        return tuple(t.shape)
    if "conv_in.weight" in sd:
        n = sum(1 for k in sd if k.startswith("body.") and k.endswith(".block1.weight") and k.count(".") == 3)
        if n == 0 or n % LEVELS:
            raise ValueError(f"adapter state dict: {n} ResNet blocks, not a positive multiple of {LEVELS} levels")
        nums_rb = n // LEVELS
        channels = tuple(shape(f"body.{i * nums_rb}.block1.weight")[0] for i in range(LEVELS))
        return "full", channels, shape("conv_in.weight")[1], nums_rb, shape("body.0.block2.weight")[-1]
    if "body.0.out_conv.weight" in sd:
        nums_rb = sum(1 for k in sd if k.startswith("body.0.body.") and k.endswith(".block1.weight"))
        channels = tuple(shape(f"body.{i}.out_conv.weight")[0] for i in range(LEVELS))
        return "light", channels, shape("body.0.in_conv.weight")[1], nums_rb, 1
    raise ValueError("adapter state dict: neither a full adapter (conv_in, body.{i}.block1/block2) nor a light one "
                     "(body.{i}.in_conv / body / out_conv)")


def pww_load_adapter(model_path: str = "synthetic:sd15:full192", device: str = "cuda:0", seed: int = 3,
                     torch_dtype: Optional[torch.dtype] = None) -> T2IAdapter:
    """A T2I-Adapter unit for `PwWSampler` / `paint_with_words(controlnet=...)`.

    `model_path` is `"synthetic:<sd15|sd21|tiny>:<full64|full192|light>"` (seeded random weights of the TencentARC v1
    shapes: sketch = full64, image / keypose = full192, color = light) or a local `.pth` state dict (read with
    `torch.load(..., weights_only=True)`), whose kind, cin, nums_rb and ksize are inferred from its keys and shapes.
    Anything else raises ValueError.  `torch_dtype` as in `pww_load_tools` (None: fp16, fp32 on mps)."""
    dtype = torch_dtype if torch_dtype is not None else (torch.float16 if device != "mps" else torch.float32)
    if model_path.startswith("synthetic:"):
        parts = model_path.split(":")
        if len(parts) != 3 or parts[1] not in _SYNTHETIC_CONFIGS or parts[2] not in _SYNTHETIC_KINDS:
            raise ValueError(f"model_path {model_path!r}: synthetic adapters are 'synthetic:<"
                             f"{'|'.join(_SYNTHETIC_CONFIGS)}>:<{'|'.join(_SYNTHETIC_KINDS)}>'")
        kind, cin, nums_rb = _SYNTHETIC_KINDS[parts[2]]
        return build_adapter(_SYNTHETIC_CONFIGS[parts[1]](), kind, cin, seed, nums_rb, dtype=dtype, device=device)
    if not model_path.endswith(".pth"):
        raise ValueError(f"model_path {model_path!r}: a 'synthetic:<config>:<kind>' name or a local .pth state dict")
    try:
        sd = torch.load(model_path, map_location="cpu", weights_only=True)
    except FileNotFoundError as e:
        raise ValueError(f"model_path {model_path!r}: no such file") from e
    if not isinstance(sd, dict):
        raise ValueError(f"{model_path}: not a state dict")
    kind, channels, cin, nums_rb, ksize = _infer(sd)
    net = T2IAdapter(kind, channels, cin, nums_rb, ksize)
    try:
        net.load_state_dict(sd, strict=True)
    except RuntimeError as e:
        raise ValueError(f"{model_path}: not a {kind} adapter of channels {channels}: {e}") from e
    net.eval().requires_grad_(False)
    net = net.to(device=device, dtype=dtype)
    if torch.device(device).type == "cuda":
        net = net.to(memory_format=torch.channels_last)
    return net
