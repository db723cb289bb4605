"""Fused channels-last UNet ops (GroupNorm[+add][+SiLU], GEGLU, add+LayerNorm) in fp16 against fp64 references to the
per-element bound of tests/unet_ops_bound.py (the full sweep is tests/test_unet_ops_bound_gpu.py), and the fused UNet
route against the plain one."""
import pytest
import torch

from paint_with_words_sd_b200 import fused_ops
from paint_with_words_sd_b200.unet import UNetConfig, build_unet
from tests import unet_ops_bound as U

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("C,HW,G", [(320, 64, 32), (640, 32, 32), (1280, 16, 32), (1280, 8, 32), (2560, 8, 32),
                                    (1920, 16, 32), (960, 32, 32), (160, 16, 8), (480, 7, 8)])
@pytest.mark.parametrize("silu,with_add", [(True, False), (True, True), (False, False)])
def test_group_norm_nhwc(C, HW, G, silu, with_add):
    g = torch.Generator().manual_seed(C + HW)
    B = 2
    x = (torch.randn(B, C, HW, HW, generator=g) * 1.5 + 0.3).half()
    gn = torch.nn.GroupNorm(G, C, eps=1e-5)
    gn.weight.data = torch.randn(C, generator=g) * 0.5 + 1.0
    gn.bias.data = torch.randn(C, generator=g) * 0.2
    add = (torch.randn(B, C, generator=g) * 0.5).half() if with_add else None
    gn_h = gn.half().cuda()
    got = fused_ops.group_norm_nhwc(x.cuda().contiguous(memory_format=torch.channels_last), gn_h,
                                    None if add is None else add.cuda(), silu=silu)
    assert got.is_contiguous(memory_format=torch.channels_last)
    # reference on the inputs as the kernel sees them (fp16 activations and affine parameters)
    ref, terms = U.gn_reference(x.cuda().flatten(2).transpose(1, 2), gn_h.weight, gn_h.bias, G, 1e-5,
                                None if add is None else add.cuda(), silu)
    U.check_within(got.flatten(2).transpose(1, 2), ref, terms, torch.float16, U.K_GN, f"gn {C} {HW} {G}")


@pytest.mark.parametrize("M,I", [(2 * 4096, 1280), (2 * 64, 5120), (3, 8), (77, 2560)])
def test_geglu(M, I):
    g = torch.Generator().manual_seed(M + I)
    h = (torch.randn(M, 2 * I, generator=g) * 2.0).half()
    ref, terms = U.geglu_reference(h)
    got = fused_ops.geglu(h.cuda()).cpu()
    U.check_within(got, ref, terms, torch.float16, U.K_GEGLU, f"geglu {M} {I}")


@pytest.mark.parametrize("M,C", [(2 * 4096, 320), (2 * 1024, 640), (2 * 256, 1280), (5, 1280), (3, 8), (7, 2048)])
@pytest.mark.parametrize("with_res", [True, False])
def test_add_layer_norm(M, C, with_res):
    g = torch.Generator().manual_seed(M + C)
    x = (torch.randn(M, C, generator=g) * 2.0).half()
    res = (torch.randn(M, C, generator=g) * 2.0).half() if with_res else None
    ln = torch.nn.LayerNorm(C)
    ln.weight.data = torch.randn(C, generator=g) * 0.5 + 1.0
    ln.bias.data = torch.randn(C, generator=g) * 0.2
    ln_h = ln.half().cuda()
    s_ref = (x.float() + res.float()).half() if with_res else x
    y_ref, terms = U.ln_reference(s_ref, ln_h.weight.cpu(), ln_h.bias.cpu(), ln.eps)
    s, y = fused_ops.add_layer_norm(x.cuda(), None if res is None else res.cuda(), ln_h)
    assert torch.equal(s.cpu(), s_ref)                      # the residual stream is bit-identical to an fp16 add
    U.check_within(y.cpu(), y_ref, terms, torch.float16, U.K_LN, f"add-layernorm {M} {C}")


def test_unet_fast_route_matches_plain_route():
    """Same fp16 weights: channels-last fused route vs the module-by-module PyTorch route (stock attention)."""
    cfg = UNetConfig.tiny()
    unet = build_unet(cfg, seed=0, dtype=torch.float16, device="cuda")
    x = torch.randn(2, 4, 16, 16, generator=torch.manual_seed(0)).cuda()
    ctx = torch.randn(2, 77, cfg.cross_attention_dim, generator=torch.manual_seed(1)).cuda().half()
    t = torch.tensor([500.0], device="cuda")
    with torch.no_grad():
        fast = unet(x, t, encoder_hidden_states=ctx).sample.float()
        orig = fused_ops.is_fast
        fused_ops.is_fast = lambda _x: False
        try:
            plain = unet(x, t, encoder_hidden_states=ctx).sample.float()
        finally:
            fused_ops.is_fast = orig
    rel = ((fast - plain).pow(2).mean().sqrt() / plain.pow(2).mean().sqrt()).item()
    assert rel < 1e-2, rel
    # leave no per-forward state behind for other tests
    from paint_with_words_sd_b200.unet import _resnets
    assert all(hasattr(r, "_pww_t") for r in _resnets(unet))
