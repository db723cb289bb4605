"""The ResNet-block fast route: conv biases folded into the time-embedding add and the native residual epilogue.

Kernel parity is bitwise against the torch statement `(a.float() + h.float() + bias).to(E)` at every ResNet shape of the
SD1.5, SD2.1 and tiny UNets; the block is compared with the plain fp32 route, also after new conv biases are loaded."""
import copy
import json
import os
import subprocess
import sys

import pytest
import torch

from paint_with_words_sd_b200 import _native, fused_ops
from paint_with_words_sd_b200.unet import UNet2DConditionModel, UNetConfig, _resnets, build_unet

pytestmark = pytest.mark.gpu

CL = torch.channels_last
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _resnet_shapes(cfg: UNetConfig):
    """Distinct (out channels, latent side, has shortcut) of the config's ResNet blocks at its sample size."""
    with torch.device("meta"):
        unet = UNet2DConditionModel(cfg)
    n = len(cfg.block_out_channels)
    levels = ([(blk, i) for i, blk in enumerate(unet.down_blocks)] + [(unet.mid_block, n - 1)]
              + [(blk, n - 1 - i) for i, blk in enumerate(unet.up_blocks)])
    shapes = set()
    for blk, level in levels:
        for r in blk.resnets:
            shapes.add((r.conv2.out_channels, cfg.sample_size >> level, r.conv_shortcut is not None))
    return sorted(shapes)


SHAPES = [(name, *s) for name, cfg in (("sd15", UNetConfig.sd15()), ("sd21", UNetConfig.sd21()),
                                       ("tiny", UNetConfig.tiny())) for s in _resnet_shapes(cfg)]


@pytest.mark.parametrize("inplace", [True, False], ids=["inplace", "out"])
@pytest.mark.parametrize("B", [2, 16])
@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16], ids=["f16", "bf16"])
@pytest.mark.parametrize("name,C,side,shortcut", SHAPES)
def test_resnet_residual_bitwise(name, C, side, shortcut, dtype, B, inplace):
    g = torch.Generator(device="cuda").manual_seed(C * 1000 + side)
    # a: the block input (identity) or the raw shortcut conv output; h: the raw conv2 output
    a = (torch.randn(B, C, side, side, generator=g, device="cuda") * (2.0 if shortcut else 4.0)).to(dtype)
    h = (torch.randn(B, C, side, side, generator=g, device="cuda") * 3.0).to(dtype)
    a, h = a.contiguous(memory_format=CL), h.contiguous(memory_format=CL)
    bias = torch.randn(C, generator=g, device="cuda") * 0.3
    ref = (a.float() + h.float() + bias[None, :, None, None]).to(dtype)
    before = _native.launch_count
    if inplace:
        out = fused_ops.resnet_residual(a, h, bias)
        assert out.data_ptr() == h.data_ptr()
    else:
        h0 = h.clone()
        out = fused_ops.resnet_residual(a, h, bias, out=torch.empty_like(h, memory_format=CL))
        assert torch.equal(h, h0)
    assert _native.launch_count - before == 1
    assert out.is_contiguous(memory_format=CL)
    assert torch.equal(out, ref)


def _blocks(dtype):
    """One shortcut block and one identity block of the tiny UNet, with the UNet's channels-last weights."""
    unet = build_unet(UNetConfig.tiny(), seed=0, dtype=dtype, device="cuda")
    res = _resnets(unet)
    return [next(r for r in res if r.conv_shortcut is not None), next(r for r in res if r.conv_shortcut is None)]


def _inputs(block, dtype, seed):
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(2, block.conv1.in_channels, 8, 8, generator=g).to("cuda", dtype).contiguous(memory_format=CL)
    temb = torch.randn(2, block.time_emb_proj.in_features, generator=g).to("cuda", dtype)
    return x, temb


def _rel(fast, plain):
    return ((fast.float() - plain).pow(2).mean().sqrt() / plain.pow(2).mean().sqrt()).item()


@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16], ids=["f16", "bf16"])
def test_fast_block_matches_plain_route_and_follows_loaded_biases(dtype):
    for k, blk in enumerate(_blocks(dtype)):
        ref = copy.deepcopy(blk).float()                    # plain fp32 route (is_fast is False for fp32)
        x, temb = _inputs(blk, dtype, k)
        with torch.no_grad():
            assert _rel(blk(x, temb), ref(x.float(), temb.float())) < 1e-2
            # new conv biases, large enough that a stale cached bias would be far off
            g = torch.Generator().manual_seed(10 + k)
            sd = {n: (torch.randn(p.shape, generator=g) * 2.0 if n.endswith("bias") and "conv" in n else p.cpu())
                  for n, p in blk.state_dict().items()}
            blk.load_state_dict(sd)
            ref.load_state_dict(sd)
            assert _rel(blk(x, temb), ref(x.float(), temb.float())) < 1e-2


def test_unet_batched_projection_follows_loaded_biases():
    """The UNet-wide time projection carries conv1's biases: a load_state_dict after a forward must rebuild it."""
    cfg = UNetConfig.tiny()
    unet = build_unet(cfg, seed=0, dtype=torch.float16, device="cuda")
    x = torch.randn(2, 4, 16, 16, generator=torch.manual_seed(0)).cuda()
    ctx = torch.randn(2, 77, cfg.cross_attention_dim, generator=torch.manual_seed(1)).cuda().half()
    t = torch.tensor([500.0], device="cuda")
    g = torch.Generator().manual_seed(3)
    with torch.no_grad():
        unet(x, t, encoder_hidden_states=ctx)
        sd = {n: (torch.randn(p.shape, generator=g) * 0.5 if n.endswith(("conv1.bias", "conv2.bias", "shortcut.bias"))
                  else p) for n, p in unet.state_dict().items()}
        unet.load_state_dict(sd)
        fast = unet(x, t, encoder_hidden_states=ctx).sample.float()
        orig = fused_ops.is_fast
        fused_ops.is_fast = lambda _x: False
        try:
            plain = unet(x, t, encoder_hidden_states=ctx).sample.float()
        finally:
            fused_ops.is_fast = orig
    assert _rel(fast, plain) < 1e-2


_LAUNCH_PROBE = """
import json, torch
from torch.profiler import ProfilerActivity, profile
from paint_with_words_sd_b200 import _native
from tests.test_resnet_residual_gpu import _blocks, _inputs
out = []
for k, blk in enumerate(_blocks(torch.float16)):
    x, temb = _inputs(blk, torch.float16, k)
    with torch.no_grad():
        object.__setattr__(blk, "_pww_t", blk.time_emb_proj(torch.nn.functional.silu(temb)))
        blk(x, temb)
        torch.cuda.synchronize()
        before = _native.launch_count
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            # CUPTI can miss the first kernels launched right after a session starts: a spin kernel goes first
            torch.cuda._sleep(20_000_000)
            torch.cuda.synchronize()
            blk(x, temb)
            torch.cuda.synchronize()
    out.append({"native": _native.launch_count - before,
                "kernels": [e.name for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA
                            and "spin_kernel" not in e.name]})
print(json.dumps(out))
"""


def test_fast_block_launches():
    """With the batched time projection present, a block is 4 GroupNorm launches + 1 residual launch around its
    convolutions, and no ATen elementwise kernel (no conv-bias pass, no separate residual add).  The profiler runs in a
    child process, so this test leaves no profiler (CUPTI) state behind in the suite's process for the other tests that
    count kernels with the profiler."""
    cmd = [sys.executable] + (["-s"] if sys.flags.no_user_site else []) + ["-c", _LAUNCH_PROBE]
    r = subprocess.run(cmd, cwd=ROOT, capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stderr[-4000:]
    blocks = json.loads(r.stdout.strip().splitlines()[-1])
    assert len(blocks) == 2
    for b in blocks:
        names = b["kernels"]
        assert b["native"] == 5
        assert sum("resnet_residual_kernel" in n for n in names) == 1, names
        assert sum("gn_stats_kernel" in n or "gn_apply_kernel" in n for n in names) == 4, names
        assert not [n for n in names if "elementwise_kernel" in n], names
