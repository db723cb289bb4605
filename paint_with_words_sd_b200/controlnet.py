"""ControlNet beside the UNet (PwW + ControlNet, the reference's `pww_controlnet` extension).

The model restates the extension's `cldm.py:118-389` (ControlNet of Zhang et al. 2023) with the blocks of `unet.py`,
under the parameter names of diffusers' `ControlNetModel`:

  * `conv_in`, `time_embedding`, `down_blocks`, `mid_block`: a copy of the UNet's encoder;
  * `controlnet_cond_embedding` (`conv_in`, `blocks.0-5`, `conv_out`): the hint block, 8 3x3 convs with SiLU between
    them taking 3 -> 16 -> 16 -> 32 -> 32 -> 96 -> 96 -> 256 -> C0 channels; three of them have stride 2, so a hint image
    at 8x the latent size lands at the latent size (cldm.py:221-237);
  * `controlnet_down_blocks.{0..11}` and `controlnet_mid_block`: the 1x1 "zero" convs (cldm.py:219, 286, 311, 353).

Forward (cldm.py:366-389): the embedded hint is added to the output of `conv_in` (`h += guided_hint`), the output of
each encoder stage goes through its zero conv and the mid-block output through `controlnet_mid_block`.  The 13 results
have exactly the shapes of the UNet's 12 skips and its mid-block output, which is where `UNet2DConditionModel.forward`
adds them (`down_block_additional_residuals`, `mid_block_additional_residual`).

The attention modules are the package's `CrossAttention` class, so `patch_unet`'s class-level patch covers them and
they run in libpww_b200; the ResNet and transformer blocks take the same fused channels-last ops as the UNet on CUDA.
"""
from __future__ import annotations

from typing import List, Optional

import torch
import torch.nn as nn
import torch.nn.functional as F

from . import fused_ops
from .unet import UNetConfig, _DownBlock, _Mid, _project_time_embeddings, timestep_embedding

HINT_CHANNELS = 3
# (in, out, stride) of the hint block's six inner convs; conv_in is 3 -> 16 and conv_out 256 -> C0
_HINT_BLOCKS = ((16, 16, 1), (16, 32, 2), (32, 32, 1), (32, 96, 2), (96, 96, 1), (96, 256, 2))


class ControlNetConditioningEmbedding(nn.Module):
    def __init__(self, out_channels: int, in_channels: int = HINT_CHANNELS):
        super().__init__()
        self.conv_in = nn.Conv2d(in_channels, _HINT_BLOCKS[0][0], 3, padding=1)
        self.blocks = nn.ModuleList([nn.Conv2d(i, o, 3, padding=1, stride=s) for i, o, s in _HINT_BLOCKS])
        self.conv_out = nn.Conv2d(_HINT_BLOCKS[-1][1], out_channels, 3, padding=1)

    def forward(self, hint):
        x = F.silu(self.conv_in(hint))
        for conv in self.blocks:
            x = F.silu(conv(x))
        return self.conv_out(x)


class ControlNetOutput:
    """diffusers' `ControlNetOutput`: `down_block_res_samples` (one per UNet skip) and `mid_block_res_sample`."""

    def __init__(self, down_block_res_samples, mid_block_res_sample):
        self.down_block_res_samples, self.mid_block_res_sample = down_block_res_samples, mid_block_res_sample

    def __iter__(self):
        return iter((self.down_block_res_samples, self.mid_block_res_sample))


class ControlNetModel(nn.Module):
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
        self.controlnet_cond_embedding = ControlNetConditioningEmbedding(ch[0])
        self.down_blocks = nn.ModuleList()
        skip_ch = [ch[0]]
        out = ch[0]
        for i, c in enumerate(ch):
            inp, out = out, c
            last = i == len(ch) - 1
            attn = None if last else (heads[i], 0, lin)
            self.down_blocks.append(_DownBlock(inp, out, temb_ch, cfg.layers_per_block, g, attn,
                                               cfg.cross_attention_dim, downsample=not last))
            skip_ch += [out] * (cfg.layers_per_block + (0 if last else 1))
        self.mid_block = _Mid(ch[-1], temb_ch, g, heads[-1], cfg.cross_attention_dim, lin)
        self.controlnet_down_blocks = nn.ModuleList([nn.Conv2d(c, c, 1) for c in skip_ch])
        self.controlnet_mid_block = nn.Conv2d(ch[-1], ch[-1], 1)

    def embed_condition(self, hint: torch.Tensor) -> torch.Tensor:
        """[R, 3, H, W] hint images in [0, 1] -> [R, C0, H/8, W/8]: the hint block alone.  It does not depend on the
        step, so a sampler embeds each image once."""
        w = self.conv_in.weight
        x = hint.to(device=w.device, dtype=w.dtype)
        if fused_ops.is_fast(x):
            x = x.contiguous(memory_format=torch.channels_last)
        return self.controlnet_cond_embedding(x)

    def forward(self, sample, timestep, encoder_hidden_states, controlnet_cond: Optional[torch.Tensor] = None,
                controlnet_cond_embedding: Optional[torch.Tensor] = None, return_dict: bool = True):
        """The 13 residuals for `sample` [B, in_channels, h, w].  Exactly one of `controlnet_cond` (hint images
        [B or 1, 3, 8h, 8w] in [0, 1]) and `controlnet_cond_embedding` (`embed_condition` of them) is given."""
        if (controlnet_cond is None) == (controlnet_cond_embedding is None):
            raise ValueError("pass exactly one of controlnet_cond and controlnet_cond_embedding")
        hint = self.embed_condition(controlnet_cond) if controlnet_cond_embedding is None else controlnet_cond_embedding
        if not torch.is_tensor(timestep):
            timestep = torch.tensor([timestep], dtype=torch.float32, device=sample.device)
        elif timestep.dim() == 0:
            timestep = timestep[None].to(sample.device)
        timestep = timestep.expand(sample.shape[0])
        wdtype = self.conv_in.weight.dtype
        temb = timestep_embedding(timestep, self.config.block_out_channels[0]).to(wdtype)
        temb = self.time_embedding["linear_2"](F.silu(self.time_embedding["linear_1"](temb)))
        x = sample.to(wdtype)
        if tuple(hint.shape[-2:]) != tuple(x.shape[-2:]):
            raise ValueError(f"the hint embeds to {tuple(hint.shape[-2:])} but the sample is {tuple(x.shape[-2:])}: "
                             "the hint image must be 8x the latent size")
        if fused_ops.is_fast(x):
            x = x.contiguous(memory_format=torch.channels_last)
            self._project_time_embeddings(temb)
        x = self.conv_in(x) + hint                       # cldm.py:379-381, h += guided_hint after the first block
        skips = [x]
        for blk in self.down_blocks:
            x, outs = blk(x, temb, encoder_hidden_states)
            skips.extend(outs)
        x = self.mid_block(x, temb, encoder_hidden_states)
        down: List[torch.Tensor] = [zc(s) for zc, s in zip(self.controlnet_down_blocks, skips)]
        mid = self.controlnet_mid_block(x)
        return ControlNetOutput(down, mid) if return_dict else (down, mid)


ControlNetModel._project_time_embeddings = _project_time_embeddings


def residual_shapes(cfg: UNetConfig, latent: int) -> List[tuple]:
    """(C, h, w) of the residuals of a ControlNet with this config at a square latent size: the UNet's skips, then its
    mid-block output."""
    ch, s = cfg.block_out_channels, latent
    shapes = [(ch[0], s, s)]
    for i, c in enumerate(ch):
        shapes += [(c, s, s)] * cfg.layers_per_block
        if i < len(ch) - 1:
            s //= 2
            shapes.append((c, s, s))
    return shapes + [(ch[-1], s, s)]


def build_controlnet(cfg: UNetConfig, seed: int = 1, dtype=torch.float32, device="cpu") -> ControlNetModel:
    """Seeded random weights for every parameter, generated on the host (then cast / moved).

    A trained ControlNet starts with its zero convs and the hint block's last conv at zero.  Here they get random
    weights like every other layer: with zeros every residual would be zero, the controlled result would equal the
    plain one, and every test comparing the two paths would pass whatever they computed."""
    with torch.random.fork_rng(devices=[]):
        torch.manual_seed(seed)
        net = ControlNetModel(cfg)
    net.eval().requires_grad_(False)
    net = net.to(device=device, dtype=dtype)
    if torch.device(device).type == "cuda":
        net = net.to(memory_format=torch.channels_last)
    return net


_SYNTHETIC_CONTROLNETS = {
    "synthetic:sd15": UNetConfig.sd15,
    "synthetic:sd21": UNetConfig.sd21,
    "synthetic:tiny": UNetConfig.tiny,
}


def pww_load_controlnet(model_path: str = "synthetic:sd15", device: str = "cuda:0", seed: int = 1,
                        torch_dtype: Optional[torch.dtype] = None) -> ControlNetModel:
    """A ControlNet for the UNet of `pww_load_tools(hf_model_path=model_path)` (or its inpaint variant: the ControlNet
    takes the 4 latent channels).  `"synthetic:<sd15|sd21|tiny>"` builds seeded random weights; there is no loader for
    trained checkpoints, and any other path raises ValueError.  `torch_dtype` as in `pww_load_tools` (None: fp16, fp32
    on mps).  The attention modules are patched like the UNet's."""
    if model_path not in _SYNTHETIC_CONTROLNETS:
        raise ValueError(f"model_path {model_path!r}: only {', '.join(_SYNTHETIC_CONTROLNETS)} ControlNets can be "
                         "built (there is no loader for trained ControlNet checkpoints)")
    from . import attention as _attention
    dtype = torch_dtype if torch_dtype is not None else (torch.float16 if device != "mps" else torch.float32)
    net = build_controlnet(_SYNTHETIC_CONTROLNETS[model_path](), seed=seed, dtype=dtype, device=device)
    _attention.patch_unet(net)
    return net
