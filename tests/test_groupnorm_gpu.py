"""The native GroupNorm (`fused_ops.group_norm_nhwc`) at every shape the UNets run: parity with fp32 F.group_norm,
precision under a large mean, bitwise determinism across calls and batch sizes, and CUDA-graph replay.

Tolerances are those of test_unet_ops_gpu.py (fp16: 4e-3 * max|ref|) and test_bf16_gpu.py (bf16: 3.2e-2)."""
import pytest
import torch
import torch.nn.functional as F

from paint_with_words_sd_b200 import fused_ops

pytestmark = pytest.mark.gpu

TOL = {torch.float16: 4e-3, torch.bfloat16: 3.2e-2}

# (HW, C, G, B)
SD15_512 = [(4096, 320, 32, 2), (4096, 640, 32, 2), (4096, 960, 32, 2),
            (1024, 320, 32, 2), (1024, 640, 32, 2), (1024, 960, 32, 2), (1024, 1280, 32, 2), (1024, 1920, 32, 2),
            (256, 640, 32, 2), (256, 1280, 32, 2), (256, 1920, 32, 2), (256, 2560, 32, 2),
            (64, 1280, 32, 2), (64, 2560, 32, 2)]
SD21_768 = [(9216, 320, 32, 2), (2304, 640, 32, 2), (576, 1280, 32, 2), (144, 2560, 32, 2)]
TINY = [(256, 160, 8, 2), (64, 480, 8, 2), (16, 960, 8, 2), (4, 640, 8, 2)]
RAGGED = [(1, 320, 32, 2), (49, 640, 32, 2), (1089, 960, 32, 2)]
BATCH = [(1024, 640, 32, 1), (256, 1280, 32, 16), (64, 2560, 32, 16)]
# 3 channels per group, one channel per group (G = 64), and wide channel slices up to one 6144-channel group
ODD = [(100, 96, 32, 2), (33, 64, 64, 3), (300, 6144, 32, 1), (16, 6144, 1, 1)]
VARIANTS = [(True, True), (True, False), (False, False)]   # (silu, with add)


def _case(HW, C, G, B, dtype, with_add, seed, offset=0.3, scale=1.5):
    g = torch.Generator().manual_seed(seed)
    x = (torch.randn(B, C, HW, generator=g) * scale + offset).to(dtype).reshape(B, C, HW, 1)
    gn = torch.nn.GroupNorm(G, C, eps=1e-5)
    gn.weight.data = torch.randn(C, generator=g) * 0.5 + 1.0
    gn.bias.data = torch.randn(C, generator=g) * 0.2
    add = (torch.randn(B, C, generator=g) * 0.5).to(dtype) if with_add else None
    return x.cuda().contiguous(memory_format=torch.channels_last), gn.to(dtype).cuda(), \
        None if add is None else add.cuda()


def _reference(x, gn, add, silu):
    """fp32 F.group_norm on the inputs as the kernel sees them (rounded activations and affine parameters)."""
    xin = x.double() + (add.double()[:, :, None, None] if add is not None else 0.0)
    ref = F.group_norm(xin, gn.num_groups, gn.weight.double(), gn.bias.double(), gn.eps)
    return (F.silu(ref) if silu else ref).float()


def _check(got, ref, dtype):
    assert got.is_contiguous(memory_format=torch.channels_last)
    err = (got.float() - ref).abs().max().item()
    bound = TOL[dtype] * max(1.0, ref.abs().max().item())
    assert err <= bound, (err, bound)


@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16], ids=["fp16", "bf16"])
@pytest.mark.parametrize("silu,with_add", VARIANTS, ids=["silu_add", "silu", "plain"])
@pytest.mark.parametrize("HW,C,G,B", SD15_512 + SD21_768 + TINY + RAGGED + BATCH + ODD)
def test_parity(HW, C, G, B, silu, with_add, dtype):
    x, gn, add = _case(HW, C, G, B, dtype, with_add, seed=HW + C + B)
    got = fused_ops.group_norm_nhwc(x, gn, add, silu=silu)
    _check(got, _reference(x, gn, add, silu), dtype)


@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16], ids=["fp16", "bf16"])
@pytest.mark.parametrize("HW,C", [(4096, 320), (1024, 640), (64, 2560)])
def test_large_mean(HW, C, dtype):
    """mean ~ 50, std ~ 1: fp32 E[x^2] - mean^2 would lose most of the variance's digits."""
    x, gn, add = _case(HW, C, 32, 2, dtype, True, seed=7, offset=50.0, scale=1.0)
    got = fused_ops.group_norm_nhwc(x, gn, add, silu=False)
    _check(got, _reference(x, gn, add, False), dtype)


@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16], ids=["fp16", "bf16"])
@pytest.mark.parametrize("HW,C,B", [(4096, 320, 2), (1024, 960, 2), (256, 1280, 16), (64, 2560, 16)])
def test_deterministic_and_batch_invariant(HW, C, B, dtype):
    x, gn, add = _case(HW, C, 32, B, dtype, True, seed=11)
    a = fused_ops.group_norm_nhwc(x, gn, add, silu=True)
    b = fused_ops.group_norm_nhwc(x, gn, add, silu=True)
    assert torch.equal(a, b)
    for i in range(B):
        one = fused_ops.group_norm_nhwc(x[i:i + 1].contiguous(memory_format=torch.channels_last), gn,
                                        add[i:i + 1].contiguous(), silu=True)
        assert torch.equal(one, a[i:i + 1]), i


@pytest.mark.parametrize("HW,C", [(4096, 320), (64, 1280)])
def test_graph_replay(HW, C):
    x, gn, add = _case(HW, C, 32, 2, torch.float16, True, seed=5)
    eager = fused_ops.group_norm_nhwc(x, gn, add, silu=True)
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        fused_ops.group_norm_nhwc(x, gn, add, silu=True)   # warm-up on the capture stream
    torch.cuda.current_stream().wait_stream(s)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        out = fused_ops.group_norm_nhwc(x, gn, add, silu=True)
    out.zero_()
    graph.replay()
    torch.cuda.synchronize()
    assert torch.equal(out, eager)
