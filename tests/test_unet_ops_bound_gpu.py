"""The native GroupNorm, GEGLU and add + LayerNorm kernels against fp64 references, per element, to the bound of
`tests/unet_ops_bound.py`: one rounding to E plus the fp32 error of each kernel's own formula.  fp16 and bf16, every
GroupNorm shape the SD1.5 / SD2.1 UNets run at 512 and 768 px, every vectors-per-lane instance of add + LayerNorm, and
the inputs where such kernels go wrong: constant groups, a std far below sqrt(eps), large means, a column slice of a
wider `add` buffer, GEGLU gates in the erf cancellation region and fp16 products that overflow.  The references are
computed on the GPU in fp64.  Each check prints `BOUND <case> worst <fraction of the allowance>` (pytest -s)."""
from types import SimpleNamespace

import pytest
import torch
import torch.nn.functional as F

from paint_with_words_sd_b200 import fused_ops
from tests import unet_ops_bound as U

pytestmark = pytest.mark.gpu
EPS = 1e-5
DT = pytest.mark.parametrize("dtype", U.DTYPES, ids=U.DTYPE_IDS)
VARIANT = pytest.mark.parametrize("silu,with_add", U.GN_VARIANTS, ids=U.GN_VARIANT_IDS)


def _report(name, worst):
    print(f"BOUND {name} worst {worst:.3f}")


# ---- GroupNorm -------------------------------------------------------------------------------------------------------
def _gn_native(x, gamma, beta, G, add, silu):
    """fused_ops.group_norm_nhwc on x [B, HW, C] (viewed as channels-last [B, C, HW, 1]); the output as [B, HW, C]."""
    B, HW, C = x.shape
    gn = SimpleNamespace(weight=gamma, bias=beta, num_groups=G, eps=EPS)
    y = fused_ops.group_norm_nhwc(x.reshape(B, HW, 1, C).permute(0, 3, 1, 2), gn, add, silu=silu)
    assert y.is_contiguous(memory_format=torch.channels_last) and y.dtype == x.dtype
    return y.permute(0, 2, 3, 1).reshape(B, HW, C)


def _gn_check(name, x, gamma, beta, G, add, silu, dtype):
    got = _gn_native(x, gamma, beta, G, add, silu)
    ref, terms = U.gn_reference(x, gamma, beta, G, EPS, add, silu)
    _report(name, U.check_within(got, ref, terms, dtype, U.K_GN, name))


@DT
@VARIANT
@pytest.mark.parametrize("HW,C,G,B", U.GN_SHAPES)
def test_groupnorm(HW, C, G, B, silu, with_add, dtype):
    x, gamma, beta, add = U.gn_inputs(HW, C, G, B, dtype, with_add, seed=HW + C + B, device="cuda")
    _gn_check(f"gn-{HW}x{C}g{G}b{B}-{silu}-{with_add}-{dtype}", x, gamma, beta, G, add, silu, dtype)


@DT
@VARIANT
@pytest.mark.parametrize("kind", ["const", "std1e-4"])
@pytest.mark.parametrize("HW,C,G,B", [(4096, 320, 32, 2), (1024, 640, 32, 3), (33, 64, 64, 1)])
def test_groupnorm_extreme_inputs(HW, C, G, B, kind, silu, with_add, dtype):
    """Constant groups (variance 0: eps alone sets rstd, and x * sc cancels sh exactly in the reference), and a std of
    1e-4 << sqrt(eps) (where an eps outside the square root would show)."""
    x, gamma, beta, add = U.gn_case_inputs(HW, C, G, B, dtype, with_add, kind, seed=HW + C, device="cuda")
    _gn_check(f"gn-{kind}-{HW}x{C}g{G}b{B}-{silu}-{with_add}-{dtype}", x, gamma, beta, G, add, silu, dtype)


@DT
@pytest.mark.parametrize("mean", [50, 1000])
@pytest.mark.parametrize("HW,C", [(4096, 320), (1024, 640), (64, 2560)])
def test_groupnorm_large_mean(HW, C, mean, dtype):
    """mean >> std: fp32 E[x^2] - mean^2 would lose most of the variance's digits; the shifted sums must not."""
    if mean == 1000 and dtype == torch.bfloat16:
        pytest.skip("bf16 spaces values near 1000 by 8: no variance left to normalise")
    x, gamma, beta, add = U.gn_case_inputs(HW, C, 32, 2, dtype, True, f"mean{mean}", seed=7, device="cuda")
    _gn_check(f"gn-mean{mean}-{HW}x{C}-{dtype}", x, gamma, beta, 32, add, False, dtype)


@DT
@pytest.mark.parametrize("silu", [True, False])
@pytest.mark.parametrize("HW,C,W,off", [(1024, 640, 4 * 1280, 1280), (64, 2560, 8960, 6400), (4096, 320, 336, 8)])
def test_groupnorm_add_column_slice(HW, C, W, off, silu, dtype):
    """add = t_all[:, off:off + C] of a wider [B, W] buffer (row stride W != C), the layout of the UNet-wide batched
    time projection; the rest of the buffer holds values that would show if the kernel read it."""
    B = 2
    x, gamma, beta, add = U.gn_inputs(HW, C, 32, B, dtype, True, seed=HW + off, device="cuda")
    wide = torch.full((B, W), 3e3 if dtype == torch.float16 else 3e5, dtype=dtype, device="cuda")
    wide[:, off:off + C] = add
    view = wide[:, off:off + C]
    assert view.stride(0) == W and view.data_ptr() % 16 == 0      # handed to the kernel as is, not copied
    _gn_check(f"gn-slice-{HW}x{C}-{W}+{off}-{silu}-{dtype}", x, gamma, beta, 32, view, silu, dtype)


# ---- GEGLU -----------------------------------------------------------------------------------------------------------
@DT
@pytest.mark.parametrize("I", U.GEGLU_I)
@pytest.mark.parametrize("M", U.GEGLU_M)
def test_geglu(M, I, dtype):
    h = U.geglu_inputs(M, I, dtype, seed=M + I, device="cuda")
    got = fused_ops.geglu(h)
    ref, terms = U.geglu_reference(h)
    name = f"geglu-{M}x{I}-{dtype}"
    _report(name, U.check_within(got, ref, terms, dtype, U.K_GEGLU, name))


@DT
def test_geglu_cancellation_matches_torch_gelu(dtype):
    """For g <= -6, 1 + erf(g / sqrt 2) is 0 in fp32 in the kernel as in torch's fp32 GELU: the product is (-)0 while
    the fp64 value is not.  A property of the formula the eager route shares, within the bound's |a| |g| term."""
    g = torch.Generator(device="cuda").manual_seed(3)
    I = 1280
    a = torch.randn(64, I, generator=g, device="cuda") * 2.0
    gate = -6.0 - torch.rand(64, I, generator=g, device="cuda") * 4.0
    h = torch.cat([a, gate], -1).to(dtype)
    got = fused_ops.geglu(h)
    assert (got == 0).all()
    assert (h[:, :I].float() * F.gelu(h[:, I:].float()) == 0).all()
    ref, terms = U.geglu_reference(h)
    assert (ref != 0).all()
    U.check_within(got, ref, terms, dtype, U.K_GEGLU, "geglu-cancellation")


def test_geglu_fp16_overflow_is_inf_like_torch():
    """Products beyond fp16's range give ±inf, at the same elements and with the same signs as torch's fp16 GEGLU."""
    g = torch.Generator(device="cuda").manual_seed(4)
    M, I = 77, 1280
    a = torch.randn(M, I, generator=g, device="cuda") * 300.0
    gate = torch.randn(M, I, generator=g, device="cuda") * 300.0
    h = torch.cat([a, gate], -1).half()
    got = fused_ops.geglu(h)
    eager = h[:, :I] * F.gelu(h[:, I:])
    ref, terms = U.geglu_reference(h)
    # away from the threshold (where the eager route's extra rounding of the GELU may decide), all three agree
    clear = (ref.abs() - 65520.0).abs() > 65520.0 * 2.0 ** -9
    over = ref.abs() >= 65520.0
    assert int((over & clear).sum()) > 1000
    for t in (got, eager):
        assert torch.equal(torch.isinf(t) & clear, over & clear)
        assert torch.equal(torch.sign(t[over & clear]).double(), torch.sign(ref[over & clear]))
    _report("geglu-overflow", U.check_within(got, ref, terms, torch.float16, U.K_GEGLU, "geglu-overflow"))


# ---- add + LayerNorm -------------------------------------------------------------------------------------------------
def _ln_check(name, x, res, gamma, beta, want_sum, dtype):
    ln = SimpleNamespace(weight=gamma, bias=beta, eps=EPS)
    s, y = fused_ops.add_layer_norm(x, res, ln, want_sum=want_sum)
    s_ref = x if res is None else x + res                   # torch's add in E: the residual stream is bit-exact
    if res is None:
        assert s is x
    elif want_sum:
        assert torch.equal(s, s_ref), name
    else:
        assert s is None
    ref, terms = U.ln_reference(s_ref, gamma, beta, EPS)
    _report(name, U.check_within(y, ref, terms, dtype, U.K_LN, name))


LN_PATHS = [(True, True), (False, True), (True, False)]        # (with res, want_sum)


@DT
@pytest.mark.parametrize("with_res,want_sum", LN_PATHS, ids=["res", "nores", "res_nosum"])
@pytest.mark.parametrize("C", U.LN_C)
@pytest.mark.parametrize("M", U.LN_M)
def test_add_layernorm(M, C, with_res, want_sum, dtype):
    x, res, gamma, beta = U.ln_inputs(M, C, dtype, seed=M + C, device="cuda")
    _ln_check(f"ln-{M}x{C}-{with_res}-{want_sum}-{dtype}", x, res if with_res else None, gamma, beta, want_sum, dtype)


@DT
@pytest.mark.parametrize("mean,std", [(100.0, 1.0), (2000.0, 20.0), (0.0, 1e-3)], ids=["mean100", "mag2000", "std1e-3"])
@pytest.mark.parametrize("C", [320, 1280, 2048])
def test_add_layernorm_large_and_flat_rows(C, mean, std, dtype):
    """A residual stream of mean 100 and std 1, fp16 magnitudes near 2000, and rows of std 1e-3 < sqrt(eps)."""
    x, res, gamma, beta = U.ln_inputs(2 * 1024, C, dtype, seed=C, device="cuda", mean=mean, std=std)
    _ln_check(f"ln-{mean:g}-{std:g}-{C}-{dtype}", x, res, gamma, beta, True, dtype)
