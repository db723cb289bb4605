"""The native GroupNorm (`fused_ops.group_norm_nhwc`): bitwise determinism across calls and batch sizes, and CUDA-graph
replay.  Its parity with fp64 at every UNet shape is tests/test_unet_ops_bound_gpu.py."""
import pytest
import torch

from paint_with_words_sd_b200 import fused_ops

pytestmark = pytest.mark.gpu


def _case(HW, C, G, B, dtype, with_add, seed):
    g = torch.Generator().manual_seed(seed)
    x = (torch.randn(B, C, HW, generator=g) * 1.5 + 0.3).to(dtype).reshape(B, C, HW, 1)
    gn = torch.nn.GroupNorm(G, C, eps=1e-5)
    gn.weight.data = torch.randn(C, generator=g) * 0.5 + 1.0
    gn.bias.data = torch.randn(C, generator=g) * 0.2
    add = (torch.randn(B, C, generator=g) * 0.5).to(dtype) if with_add else None
    return x.cuda().contiguous(memory_format=torch.channels_last), gn.to(dtype).cuda(), \
        None if add is None else add.cuda()


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
