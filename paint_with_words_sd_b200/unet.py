"""Stable-Diffusion-shaped UNet with the diffusers-0.10.0 `UNet2DConditionModel` module contract.

This is the CALLER of the hot path (SURVEY.md 8f-1), not the product: diffusers is not installed and
there are no weights on disk, so the architecture is restated from its published description
(hyper-parameters cross-checked with pww_controlnet/models/cldm_v15.yaml:38-53 and cldm_v21.yaml:39-55
in the reference) and filled with seeded random weights.  What matters for the drop-in boundary:

  * attention modules are instances of a class literally named `CrossAttention` exposing
    `to_q/to_k/to_v` (Linear, no bias), `to_out = ModuleList([Linear, Dropout])`, `heads`, `scale`,
    `reshape_heads_to_batch_dim`, `reshape_batch_dim_to_heads`  -- the attributes the reference's
    `inj_forward` touches (paint_with_words.py:76-85, 112-123);
  * `BasicTransformerBlock` hands whatever was passed as `encoder_hidden_states` (a Tensor or the PwW
    context dict) to `attn2` untouched, which is what lets the dict travel (paint_with_words.py:483-487);
  * `unet(x, t, encoder_hidden_states=...)` returns an object with `.sample`; `unet.in_channels` exists.

The stock `CrossAttention.forward` below is plain PyTorch attention (what diffusers does before the
reference monkey-patches `__call__`, paint_with_words.py:193-195).
"""
from __future__ import annotations

import math
from dataclasses import dataclass, field
from typing import List, Optional, Sequence, Tuple, Union

import torch
import torch.nn as nn
import torch.nn.functional as F

from . import fused_ops


@dataclass
class UNetConfig:
    in_channels: int = 4
    out_channels: int = 4
    block_out_channels: Tuple[int, ...] = (320, 640, 1280, 1280)
    layers_per_block: int = 2
    cross_attention_dim: int = 768
    attention_heads: Union[int, Tuple[int, ...]] = 8          # diffusers' "attention_head_dim" (really head count)
    use_linear_projection: bool = False
    norm_num_groups: int = 32
    sample_size: int = 64

    @staticmethod
    def sd15(in_channels: int = 4) -> "UNetConfig":
        return UNetConfig(in_channels=in_channels)

    @staticmethod
    def sd15_inpaint() -> "UNetConfig":
        return UNetConfig(in_channels=9)

    @staticmethod
    def sd21() -> "UNetConfig":
        return UNetConfig(cross_attention_dim=1024, attention_heads=(5, 10, 20, 20),
                          use_linear_projection=True, sample_size=96)

    @staticmethod
    def tiny(in_channels: int = 4) -> "UNetConfig":
        """Same topology at half width with 4 heads (head dims 40/80/160/160 -- inside the kernel family):
        for CPU tests and the smoke run."""
        return UNetConfig(in_channels=in_channels, block_out_channels=(160, 320, 640, 640), cross_attention_dim=64,
                          attention_heads=4, norm_num_groups=8, sample_size=16)


class CrossAttention(nn.Module):
    def __init__(self, query_dim: int, cross_attention_dim: Optional[int] = None, heads: int = 8,
                 dim_head: int = 64, dropout: float = 0.0):
        super().__init__()
        inner = dim_head * heads
        cross_attention_dim = cross_attention_dim if cross_attention_dim is not None else query_dim
        self.scale = dim_head ** -0.5
        self.heads = heads
        self.to_q = nn.Linear(query_dim, inner, bias=False)
        self.to_k = nn.Linear(cross_attention_dim, inner, bias=False)
        self.to_v = nn.Linear(cross_attention_dim, inner, bias=False)
        self.to_out = nn.ModuleList([nn.Linear(inner, query_dim), nn.Dropout(dropout)])

    def reshape_heads_to_batch_dim(self, t):
        b, n, c = t.shape
        h = self.heads
        return t.reshape(b, n, h, c // h).permute(0, 2, 1, 3).reshape(b * h, n, c // h)

    def reshape_batch_dim_to_heads(self, t):
        bh, n, d = t.shape
        h = self.heads
        return t.reshape(bh // h, h, n, d).permute(0, 2, 1, 3).reshape(bh // h, n, d * h)

    def forward(self, hidden_states, context=None, mask=None):
        ctx = hidden_states if context is None else context
        q = self.reshape_heads_to_batch_dim(self.to_q(hidden_states))
        k = self.reshape_heads_to_batch_dim(self.to_k(ctx))
        v = self.reshape_heads_to_batch_dim(self.to_v(ctx))
        p = (torch.matmul(q, k.transpose(-1, -2)) * self.scale).softmax(dim=-1)
        o = self.reshape_batch_dim_to_heads(torch.matmul(p.to(v.dtype), v))
        return self.to_out[1](self.to_out[0](o))


class GEGLU(nn.Module):
    def __init__(self, dim_in, dim_out):
        super().__init__()
        self.proj = nn.Linear(dim_in, dim_out * 2)

    def forward(self, x):
        h = self.proj(x)
        if fused_ops.is_fast(h):
            return fused_ops.geglu(h)              # one launch instead of chunk + gelu + mul
        x, gate = h.chunk(2, dim=-1)
        return x * F.gelu(gate)


class FeedForward(nn.Module):
    def __init__(self, dim, mult=4):
        super().__init__()
        self.net = nn.ModuleList([GEGLU(dim, dim * mult), nn.Dropout(0.0), nn.Linear(dim * mult, dim)])

    def forward(self, x):
        for m in self.net:
            x = m(x)
        return x


class BasicTransformerBlock(nn.Module):
    def __init__(self, dim, heads, dim_head, cross_attention_dim):
        super().__init__()
        self.attn1 = CrossAttention(dim, None, heads, dim_head)
        self.ff = FeedForward(dim)
        self.attn2 = CrossAttention(dim, cross_attention_dim, heads, dim_head)
        self.norm1, self.norm2, self.norm3 = nn.LayerNorm(dim), nn.LayerNorm(dim), nn.LayerNorm(dim)

    def forward(self, x, context=None):
        if fused_ops.is_fast(x):
            # residual add fused into the following LayerNorm: 3 LN launches + 1 add instead of 3 LN + 3 adds
            _, h = fused_ops.add_layer_norm(x, None, self.norm1)
            x, h = fused_ops.add_layer_norm(self.attn1(h), x, self.norm2)
            x, h = fused_ops.add_layer_norm(self.attn2(h, context=context), x, self.norm3)
            return self.ff(h) + x
        x = self.attn1(self.norm1(x)) + x
        x = self.attn2(self.norm2(x), context=context) + x
        return self.ff(self.norm3(x)) + x


class Transformer2DModel(nn.Module):
    def __init__(self, heads, dim_head, in_channels, cross_attention_dim, groups, linear_proj):
        super().__init__()
        inner = heads * dim_head
        self.linear_proj = linear_proj
        self.norm = nn.GroupNorm(groups, in_channels, eps=1e-6)
        self.proj_in = nn.Linear(in_channels, inner) if linear_proj else nn.Conv2d(in_channels, inner, 1)
        self.transformer_blocks = nn.ModuleList([BasicTransformerBlock(inner, heads, dim_head, cross_attention_dim)])
        self.proj_out = nn.Linear(inner, in_channels) if linear_proj else nn.Conv2d(inner, in_channels, 1)

    def _forward_fast(self, x, encoder_hidden_states):
        """Channels-last route: the token view [B,HW,C] of an NHWC activation is free, so GroupNorm is one fused
        launch and the 1x1 projections are plain GEMMs -- no layout conversion anywhere."""
        b, c, h, w = x.shape
        if not x.is_contiguous(memory_format=torch.channels_last):
            x = x.contiguous(memory_format=torch.channels_last)
        res = x.permute(0, 2, 3, 1).reshape(b, h * w, c)           # token view of the NHWC activation (no copy)
        t = fused_ops.group_norm_nhwc(x, self.norm, silu=False).permute(0, 2, 3, 1).reshape(b, h * w, c)
        wi = self.proj_in.weight
        t = F.linear(t, wi.reshape(wi.shape[0], wi.shape[1]), self.proj_in.bias)
        for blk in self.transformer_blocks:
            t = blk(t, context=encoder_hidden_states)
        wo = self.proj_out.weight
        t = F.linear(t, wo.reshape(wo.shape[0], wo.shape[1]), self.proj_out.bias) + res   # contiguous, vectorised add
        return t.reshape(b, h, w, c).permute(0, 3, 1, 2)

    def forward(self, x, encoder_hidden_states=None):
        if fused_ops.is_fast(x):
            return self._forward_fast(x, encoder_hidden_states)
        b, c, h, w = x.shape
        res = x
        x = self.norm(x)
        if self.linear_proj:
            x = self.proj_in(x.permute(0, 2, 3, 1).reshape(b, h * w, c))
        else:
            x = self.proj_in(x).permute(0, 2, 3, 1).reshape(b, h * w, -1)
        for blk in self.transformer_blocks:
            x = blk(x, context=encoder_hidden_states)
        if self.linear_proj:
            x = self.proj_out(x).reshape(b, h, w, c).permute(0, 3, 1, 2)
        else:
            x = self.proj_out(x.reshape(b, h, w, -1).permute(0, 3, 1, 2))
        return x + res


class ResnetBlock2D(nn.Module):
    def __init__(self, in_ch, out_ch, temb_ch, groups):
        super().__init__()
        self.norm1 = nn.GroupNorm(groups, in_ch, eps=1e-5)
        self.conv1 = nn.Conv2d(in_ch, out_ch, 3, padding=1)
        self.time_emb_proj = nn.Linear(temb_ch, out_ch)
        self.norm2 = nn.GroupNorm(groups, out_ch, eps=1e-5)
        self.conv2 = nn.Conv2d(out_ch, out_ch, 3, padding=1)
        self.conv_shortcut = nn.Conv2d(in_ch, out_ch, 1) if in_ch != out_ch else None

    def forward(self, x, temb):
        if fused_ops.is_fast(x):
            # GroupNorm+SiLU fused; the convolutions run without bias, so no per-channel bias pass touches their outputs:
            # conv1's bias rides with the time embedding into the second GroupNorm's add, conv2's and the shortcut's go
            # into the residual epilogue
            t_bias, res_bias = _block_biases(self)
            h = self.conv1._conv_forward(fused_ops.group_norm_nhwc(x, self.norm1, silu=True), self.conv1.weight, None)
            t = getattr(self, "_pww_t", None)       # slice of the UNet-wide batched projection, when provided
            if t is None:
                t = F.linear(F.silu(temb), self.time_emb_proj.weight, t_bias)
            h = self.conv2._conv_forward(fused_ops.group_norm_nhwc(h, self.norm2, add=t, silu=True), self.conv2.weight,
                                         None)
            sc = self.conv_shortcut
            a = x if sc is None else sc._conv_forward(x, sc.weight, None)
            return fused_ops.resnet_residual(a, h, res_bias)
        h = self.conv1(F.silu(self.norm1(x)))
        h = h + self.time_emb_proj(F.silu(temb))[:, :, None, None]
        h = self.conv2(F.silu(self.norm2(h)))
        return (x if self.conv_shortcut is None else self.conv_shortcut(x)) + h


class Downsample2D(nn.Module):
    def __init__(self, ch):
        super().__init__()
        self.conv = nn.Conv2d(ch, ch, 3, stride=2, padding=1)

    def forward(self, x):
        return self.conv(x)


class Upsample2D(nn.Module):
    def __init__(self, ch):
        super().__init__()
        self.conv = nn.Conv2d(ch, ch, 3, padding=1)

    def forward(self, x):
        return self.conv(F.interpolate(x, scale_factor=2.0, mode="nearest"))


class _DownBlock(nn.Module):
    def __init__(self, in_ch, out_ch, temb_ch, n_layers, groups, attn: Optional[Tuple[int, int, bool]], cross_dim,
                 downsample: bool):
        super().__init__()
        self.resnets = nn.ModuleList([ResnetBlock2D(in_ch if i == 0 else out_ch, out_ch, temb_ch, groups)
                                      for i in range(n_layers)])
        self.attentions = None
        if attn is not None:
            heads, _, lin = attn
            self.attentions = nn.ModuleList([Transformer2DModel(heads, out_ch // heads, out_ch, cross_dim, groups, lin)
                                             for _ in range(n_layers)])
        self.downsamplers = nn.ModuleList([Downsample2D(out_ch)]) if downsample else None

    def forward(self, x, temb, ctx):
        outs = []
        for i, res in enumerate(self.resnets):
            x = res(x, temb)
            if self.attentions is not None:
                x = self.attentions[i](x, ctx)
            outs.append(x)
        if self.downsamplers is not None:
            x = self.downsamplers[0](x)
            outs.append(x)
        return x, outs


class _UpBlock(nn.Module):
    def __init__(self, in_ch, out_ch, prev_ch, temb_ch, n_layers, groups, attn, cross_dim, upsample: bool):
        super().__init__()
        res = []
        for i in range(n_layers):
            skip = in_ch if i == n_layers - 1 else out_ch
            res.append(ResnetBlock2D((prev_ch if i == 0 else out_ch) + skip, out_ch, temb_ch, groups))
        self.resnets = nn.ModuleList(res)
        self.attentions = None
        if attn is not None:
            heads, _, lin = attn
            self.attentions = nn.ModuleList([Transformer2DModel(heads, out_ch // heads, out_ch, cross_dim, groups, lin)
                                             for _ in range(n_layers)])
        self.upsamplers = nn.ModuleList([Upsample2D(out_ch)]) if upsample else None

    def forward(self, x, skips: List[torch.Tensor], temb, ctx):
        for i, res in enumerate(self.resnets):
            x = res(torch.cat([x, skips.pop()], dim=1), temb)
            if self.attentions is not None:
                x = self.attentions[i](x, ctx)
        if self.upsamplers is not None:
            x = self.upsamplers[0](x)
        return x


class _Mid(nn.Module):
    def __init__(self, ch, temb_ch, groups, heads, cross_dim, lin):
        super().__init__()
        self.resnets = nn.ModuleList([ResnetBlock2D(ch, ch, temb_ch, groups), ResnetBlock2D(ch, ch, temb_ch, groups)])
        self.attentions = nn.ModuleList([Transformer2DModel(heads, ch // heads, ch, cross_dim, groups, lin)])

    def forward(self, x, temb, ctx):
        x = self.resnets[0](x, temb)
        x = self.attentions[0](x, ctx)
        return self.resnets[1](x, temb)


class _Sample:
    def __init__(self, sample):
        self.sample = sample


def timestep_embedding(t: torch.Tensor, dim: int) -> torch.Tensor:
    """Sinusoidal embedding, flip_sin_to_cos=True, downscale_freq_shift=0 (SD UNet settings)."""
    half = dim // 2
    freqs = torch.exp(-math.log(10000.0) * torch.arange(half, dtype=torch.float32, device=t.device) / half)
    ang = t.float()[:, None] * freqs[None]
    return torch.cat([torch.cos(ang), torch.sin(ang)], dim=-1)


class UNet2DConditionModel(nn.Module):
    def __init__(self, cfg: UNetConfig = UNetConfig()):
        super().__init__()
        self.config = cfg
        self.in_channels = cfg.in_channels
        ch = cfg.block_out_channels
        temb_ch = ch[0] * 4
        g = cfg.norm_num_groups
        heads = cfg.attention_heads if isinstance(cfg.attention_heads, (tuple, list)) else (cfg.attention_heads,) * len(ch)
        lin = cfg.use_linear_projection
        self.conv_in = nn.Conv2d(cfg.in_channels, ch[0], 3, padding=1)
        self.time_embedding = nn.ModuleDict({"linear_1": nn.Linear(ch[0], temb_ch), "linear_2": nn.Linear(temb_ch, temb_ch)})
        self.down_blocks = nn.ModuleList()
        out = ch[0]
        for i, c in enumerate(ch):
            inp, out = out, c
            last = i == len(ch) - 1
            attn = None if last else (heads[i], 0, lin)
            self.down_blocks.append(_DownBlock(inp, out, temb_ch, cfg.layers_per_block, g, attn,
                                               cfg.cross_attention_dim, downsample=not last))
        self.mid_block = _Mid(ch[-1], temb_ch, g, heads[-1], cfg.cross_attention_dim, lin)
        self.up_blocks = nn.ModuleList()
        rev, rheads = list(reversed(ch)), list(reversed(heads))
        out = rev[0]
        for i, c in enumerate(rev):
            prev, out = out, c
            inp = rev[min(i + 1, len(ch) - 1)]
            last = i == len(ch) - 1
            attn = None if i == 0 else (rheads[i], 0, lin)
            self.up_blocks.append(_UpBlock(inp, out, prev, temb_ch, cfg.layers_per_block + 1, g, attn,
                                           cfg.cross_attention_dim, upsample=not last))
        self.conv_norm_out = nn.GroupNorm(g, ch[0], eps=1e-5)
        self.conv_out = nn.Conv2d(ch[0], cfg.out_channels, 3, padding=1)

    def forward(self, sample, timestep, encoder_hidden_states=None, down_block_additional_residuals=None,
                mid_block_additional_residual=None):
        """`down_block_additional_residuals` (one per skip) and `mid_block_additional_residual` are a ControlNet's
        outputs, as in diffusers: residual k is added to skip k before the decoder concatenates it, the mid residual to
        the mid-block output.  Residuals of fewer images than the batch go into its first images (guess mode: the cond
        half).  A context dict may carry "CONTROL_SCALES", an fp32 [len(skips) + 1, rows] device tensor: residual k of
        image b is multiplied by CONTROL_SCALES[k, b] first (absent: 1, diffusers' plain add)."""
        if (down_block_additional_residuals is None) != (mid_block_additional_residual is None):
            raise ValueError("down_block_additional_residuals and mid_block_additional_residual go together")
        if not torch.is_tensor(timestep):
            timestep = torch.tensor([timestep], dtype=torch.float32, device=sample.device)
        elif timestep.dim() == 0:
            timestep = timestep[None].to(sample.device)
        timestep = timestep.expand(sample.shape[0])
        wdtype = self.conv_in.weight.dtype
        temb = timestep_embedding(timestep, self.config.block_out_channels[0]).to(wdtype)
        temb = self.time_embedding["linear_2"](F.silu(self.time_embedding["linear_1"](temb)))
        x = sample.to(wdtype)
        fast = fused_ops.is_fast(x)
        if fast:
            x = x.contiguous(memory_format=torch.channels_last)
            self._project_time_embeddings(temb)
        x = self.conv_in(x)
        skips = [x]
        for blk in self.down_blocks:
            x, outs = blk(x, temb, encoder_hidden_states)
            skips.extend(outs)
        x = self.mid_block(x, temb, encoder_hidden_states)
        if mid_block_additional_residual is not None:
            residuals = list(down_block_additional_residuals) + [mid_block_additional_residual]
            if len(residuals) != len(skips) + 1:
                raise ValueError(f"{len(residuals) - 1} down-block residuals for {len(skips)} skips")
            scales = encoder_hidden_states.get("CONTROL_SCALES") if isinstance(encoder_hidden_states, dict) else None
            if fast:
                fused_ops.control_inject(skips + [x], residuals, scales)   # one launch, in place
            else:
                *skips, x = add_control_residuals(skips + [x], residuals, scales)
        for blk in self.up_blocks:
            x = blk(x, skips, temb, encoder_hidden_states)
        if fast:
            x = self.conv_out(fused_ops.group_norm_nhwc(x, self.conv_norm_out, silu=True))
        else:
            x = self.conv_out(F.silu(self.conv_norm_out(x)))
        return _Sample(x)


def add_control_residuals(targets: Sequence[torch.Tensor], residuals: Sequence[torch.Tensor],
                          scales: Optional[torch.Tensor] = None) -> List[torch.Tensor]:
    """The torch statement of `pww_control_inject`: target_k[:rows] + (residual_k * scales[k]) with the product
    rounded to the target's type (rows = residual_k.shape[0]; scales an fp32 [n, rows] tensor or None for 1)."""
    out = []
    for k, (d, r) in enumerate(zip(targets, residuals)):
        rows = r.shape[0]
        if tuple(r.shape[1:]) != tuple(d.shape[1:]) or rows > d.shape[0]:
            raise ValueError(f"residual {k} {tuple(r.shape)} does not match its target {tuple(d.shape)}")
        p = r if scales is None else r * scales[k].to(r.device).view(rows, 1, 1, 1)
        p = p.to(d.dtype)
        out.append(d + p if rows == d.shape[0] else torch.cat([d[:rows] + p, d[rows:]], 0))
    return out


def combine_control_residuals(res_per_unit: Sequence[Sequence[torch.Tensor]], scales: torch.Tensor) -> List[torch.Tensor]:
    """The torch statement of `pww_control_combine`: level k is (res_0k * s[0, k]).to(E) + (res_1k * s[1, k]).to(E) +
    ..., summed left to right in the residuals' type E (scales an fp32 [units, n, rows] tensor)."""
    out = []
    for k in range(len(res_per_unit[0])):
        total = None
        for u, unit in enumerate(res_per_unit):
            r = unit[k]
            p = (r * scales[u, k].to(r.device).view(r.shape[0], 1, 1, 1)).to(r.dtype)
            total = p if total is None else total + p
        out.append(total)
    return out


def _resnets(unet: nn.Module):
    return [m for m in unet.modules() if isinstance(m, ResnetBlock2D)]


def _param_key(params) -> tuple:
    """Cache key of tensors derived from `params`: their storage and version counters, so an in-place update
    (load_state_dict, a weight broadcast after a first forward) invalidates the derived tensors."""
    return tuple((p.data_ptr(), p._version, p.dtype, p.device) for p in params)


def _block_biases(block: ResnetBlock2D):
    """The fast route's biases of one ResNet block: (time_emb_proj.bias + conv1.bias in the parameters' type, the
    time-embedding projection's bias; conv2.bias + conv_shortcut.bias in fp32, the residual epilogue's).  Each sum is
    taken in fp32 and rounded once; both are cached on the block, keyed on the biases' storage and version counters."""
    sc = block.conv_shortcut
    params = [block.time_emb_proj.bias, block.conv1.bias, block.conv2.bias] + ([] if sc is None else [sc.bias])
    key = _param_key(params)
    hit = block.__dict__.get("_pww_biases")
    if hit is None or hit[0] != key:
        tb = block.time_emb_proj.bias.float() + block.conv1.bias.float()
        rb = block.conv2.bias.float() + (0.0 if sc is None else sc.bias.float())
        hit = (key, tb.to(block.time_emb_proj.bias.dtype).detach(), rb.detach().contiguous())
        block.__dict__["_pww_biases"] = hit
    return hit[1], hit[2]


def _project_time_embeddings(self, temb):
    """All 22 ResNet `time_emb_proj(silu(temb))` projections as ONE GEMM, each block's conv1 bias folded into its
    projection bias (`_block_biases`); each block reads its column slice.  The concatenated weights and biases are
    cached, keyed on the parameters' storage and version counters."""
    res = _resnets(self)
    key = _param_key([p for r in res for p in (r.time_emb_proj.weight, r.time_emb_proj.bias, r.conv1.bias)])
    cache = self.__dict__.get("_pww_temb_w")
    if cache is None or cache[0] != key:
        w = torch.cat([r.time_emb_proj.weight for r in res], 0).detach().contiguous()
        b = torch.cat([_block_biases(r)[0] for r in res], 0).contiguous()
        cache = (key, w, b)
        self.__dict__["_pww_temb_w"] = cache
    t_all = F.linear(F.silu(temb), cache[1], cache[2])
    off = 0
    for r in res:
        n = r.time_emb_proj.weight.shape[0]
        object.__setattr__(r, "_pww_t", t_all[:, off:off + n])
        off += n


UNet2DConditionModel._project_time_embeddings = _project_time_embeddings


def attention_modules(unet: nn.Module):
    return [m for m in unet.modules() if m.__class__.__name__ == "CrossAttention"]


def build_unet(cfg: UNetConfig, seed: int = 0, dtype=torch.float32, device="cpu") -> UNet2DConditionModel:
    """Seeded random weights, generated on the host so every rank / both bench arms get identical
    parameters (then cast / moved)."""
    with torch.random.fork_rng(devices=[]):
        torch.manual_seed(seed)
        unet = UNet2DConditionModel(cfg)
    unet.eval().requires_grad_(False)
    unet = unet.to(device=device, dtype=dtype)
    if torch.device(device).type == "cuda":
        unet = unet.to(memory_format=torch.channels_last)      # NHWC conv weights: no layout conversion kernels
    return unet
