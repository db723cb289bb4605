"""GPU parity of the self-attention kernel (pww_attn_fwd_f16, context=None path of inj_forward) against the oracle."""
import pytest
import torch

from oracle import pww_oracle as O
from paint_with_words_sd_b200 import _native
from paint_with_words_sd_b200 import attention as A

pytestmark = pytest.mark.gpu

SHAPES = [(4096, 8, 40), (1024, 8, 80), (256, 8, 160), (64, 8, 160), (16, 8, 160),       # SD1.5 512^2 / 256^2
          (2304, 10, 64), (576, 20, 64), (144, 20, 64),                                   # SD2.1 768^2 (9216 below)
          (100, 2, 40), (129, 3, 80), (333, 1, 160), (1, 2, 64), (200, 4, 64), (257, 2, 40)]  # ragged


def _qkv(B, N, H, D, seed, spread=0.5):
    g = torch.Generator().manual_seed(seed)
    C = H * D
    return [(torch.randn(B, N, C, generator=g) * spread).half() for _ in range(3)]


def _native_attention(q, k, v, H, scale):
    """The library's own kernel at every size (the shim's default picks per size)."""
    old = A.SELF_ATTN_IMPL
    A.SELF_ATTN_IMPL = "native"
    try:
        before = _native.launch_count
        out = A.self_attention(q, k, v, H, scale)
        assert _native.launch_count == before + 1
    finally:
        A.SELF_ATTN_IMPL = old
    return out


def _check(q, k, v, H, D, tol=2e-3):
    scale = D ** -0.5
    got = _native_attention(q.cuda(), k.cuda(), v.cuda(), H, scale)
    torch.cuda.synchronize()
    got = got.float().cpu()
    ref = torch.cat([O.attention_core(q[b:b + 1].float(), k[b:b + 1].float(), v[b:b + 1].float(), H, scale)
                     for b in range(q.shape[0])], 0)
    err = (got - ref).abs().max().item() / ref.abs().max().item()
    assert err <= tol, err


@pytest.mark.parametrize("N,H,D", SHAPES)
def test_self_attention_matches_oracle(N, H, D):
    q, k, v = _qkv(2 if N <= 1024 else 1, N, H, D, seed=N + D)
    _check(q, k, v, H, D)


def test_self_attention_sd21_top_level():
    q, k, v = _qkv(1, 9216, 5, 64, seed=9)
    _check(q, k, v, 5, 64)


def test_peaky_scores_exercise_the_rescale_path():
    """Large, growing logits force the running maximum to move by more than the lazy-rescale threshold."""
    N, H, D = 512, 2, 64
    q, k, v = _qkv(1, N, H, D, seed=1, spread=0.5)
    k = k.float()
    k *= torch.linspace(0.2, 6.0, N)[None, :, None]          # later key tiles carry much larger scores
    _check(q, k.half(), v, H, D, tol=3e-3)


def test_strided_qkv_views():
    """q/k/v as column slices of one fused [B,N,3C] buffer (shared row stride 3C)."""
    N, H, D = 256, 8, 40
    C = H * D
    q, k, v = _qkv(1, N, H, D, seed=3)
    fused = torch.cat([q, k, v], -1).cuda()
    got = _native_attention(fused[..., :C], fused[..., C:2 * C], fused[..., 2 * C:], H, D ** -0.5).float().cpu()
    ref = O.attention_core(q.float(), k.float(), v.float(), H, D ** -0.5)
    assert (got - ref).abs().max().item() <= 2e-3 * ref.abs().max().item()


def test_default_dispatch_matches_oracle_on_both_sides_of_the_switch():
    """The shim's default: native kernel up to SELF_ATTN_NATIVE_MAX_KEYS keys, torch's library attention above -- same
    numbers either way."""
    switch = A.SELF_ATTN_NATIVE_MAX_KEYS
    for N, native in ((switch // 4, True), (2 * switch, False)):
        q, k, v = _qkv(1, N, 8, 40, seed=N)
        before = _native.launch_count
        got = A.self_attention(q.cuda(), k.cuda(), v.cuda(), 8, 40 ** -0.5).float().cpu()
        assert (_native.launch_count == before + 1) == native
        ref = O.attention_core(q.float(), k.float(), v.float(), 8, 40 ** -0.5)
        assert (got - ref).abs().max().item() <= 2e-3 * ref.abs().max().item()
