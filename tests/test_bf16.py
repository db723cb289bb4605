"""bf16 without a GPU: every `_bf16` entry point validates its arguments exactly like its `_f16` twin (before any CUDA
call), the sampler entry points take the bf16 dtype code, and the public API builds bf16 models on request."""
import ctypes

import pytest
import torch

from paint_with_words_sd_b200 import _native
from paint_with_words_sd_b200 import pipeline as PL

BF16_ENTRY_POINTS = ("pww_xattn_stats", "pww_xattn_fwd", "pww_xattn_fused", "pww_xattn_stats_multi",
                     "pww_xattn_fwd_multi", "pww_xattn_fused_multi", "pww_attn_fwd", "pww_groupnorm_nhwc",
                     "pww_geglu", "pww_add_layernorm")


@pytest.fixture(scope="module")
def buf16():
    buf = (ctypes.c_char * 8192)()
    return buf, (ctypes.addressof(buf) + 15) // 16 * 16


def _cases(name, p):
    """{case: argument tuple} of `name` for a null pointer, a misaligned pointer and, where the call has them, head dim
    48 and T = 200 (or an unsupported channel count); every case fails validation before any CUDA call."""
    H, N = 8, 64

    def xattn(q=p, D=40, T=77):
        C = H * D
        if name in ("pww_xattn_stats", "pww_xattn_stats_multi"):
            return (q, p, 1, H, N, T, D, N * C, C, T * C, C, 0 if name == "pww_xattn_stats" else p, None, p, p, 8, None)
        if name in ("pww_xattn_fwd", "pww_xattn_fwd_multi"):
            return (q, p, p, p, 1, H, N, T, D, N * C, C, T * C, C, N * C, C, None, 0, None, None, None, 0.158, None)
        return (q, p, p, p, 1, H, N, T, D, N * C, C, T * C, C, N * C, C, p, N * 32, 1, p, None,
                0 if name == "pww_xattn_fused" else p, p, 0.158, p, p, 8, None)

    if name.startswith("pww_xattn"):
        return {"null": xattn(q=None), "misaligned": xattn(q=p + 2), "head_dim_48": xattn(D=48),
                "T_200": xattn(T=200)}
    if name == "pww_attn_fwd":
        a = lambda q=p, D=40: (q, p, p, p, 1, H, N, D, N * H * D, H * D, N * H * D, H * D, 0.158, None)  # noqa: E731
        return {"null": a(q=None), "misaligned": a(q=p + 2), "head_dim_48": a(D=48)}
    if name == "pww_groupnorm_nhwc":
        g = lambda x=p, C=64, G=32: (x, None, 0, p, p, p, 1, 16, C, G, 1e-5, 1, p, 4096, None)  # noqa: E731
        return {"null": g(x=None), "misaligned": g(x=p + 2), "channels_12": g(C=12, G=4), "groups_128": g(C=256, G=128)}
    if name == "pww_geglu":
        return {"null": (None, p, 4, 64, None), "misaligned": (p + 2, p, 4, 64, None), "width_12": (p, p, 4, 12, None)}
    assert name == "pww_add_layernorm"
    ln = lambda x=p, C=64: (x, None, p, p, None, p, 4, C, 1e-5, None)  # noqa: E731
    return {"null": ln(x=None), "misaligned": ln(x=p + 2), "channels_12": ln(C=12), "channels_4096": ln(C=4096)}


@pytest.mark.parametrize("name", BF16_ENTRY_POINTS)
def test_bf16_entry_points_validate_like_their_f16_twins(name, buf16):
    L = _native.lib()
    _, p = buf16
    for case, args in _cases(name, p).items():
        f16 = getattr(L, name + "_f16")(*args)
        bf16 = getattr(L, name + "_bf16")(*args)
        assert f16 in (-1, -2, -4), (case, f16)         # the case really fails validation
        assert bf16 == f16, (name, case, f16, bf16)


def test_bf16_symbols_take_their_twins_signatures():
    L = _native.lib()
    for name in BF16_ENTRY_POINTS:
        f16, bf16 = getattr(L, name + "_f16"), getattr(L, name + "_bf16")
        assert bf16.argtypes == f16.argtypes and bf16.restype == f16.restype, name
        assert name + "_bf16" in _native.EXPORTS


def test_sampler_entry_points_take_the_bf16_code(buf16):
    """The bf16 code (4) goes through the same argument checks as fp16; the unassigned codes 2 and 3 still return
    PWW_ERR_UNSUPPORTED before any CUDA call, as they did before bf16."""
    L = _native.lib()
    _, p = buf16
    F16, BF16 = _native.PWW_DTYPE_F16, _native.PWW_DTYPE_BF16
    assert BF16 == 4
    inp = lambda lat=p, scale=p, extra=None, out=p, dt=F16, m=1, c=4, h=8, w=8: L.pww_sampler_input(  # noqa: E731
        lat, scale, extra, out, dt, m, c, h, w, None)
    for dt in (F16, BF16):
        assert inp(lat=None, dt=dt) == -1 and inp(scale=None, dt=dt) == -1 and inp(out=None, dt=dt) == -1
        assert inp(m=0, dt=dt) == -1 and inp(h=0, dt=dt) == -1 and inp(w=-2, dt=dt) == -1
        assert inp(c=5, dt=dt) == -1 and inp(c=9, dt=dt) == -1 and inp(extra=p, dt=dt) == -1
    assert inp(dt=2) == -2 and inp(dt=3) == -2 and inp(dt=5) == -2 and inp(dt=-1, c=9, extra=p) == -2
    upd = lambda eps=p, dt=F16, lat=p, hist=p, hl=4, noise=None, gs=p, beta=p, form=p, m=2, h=8, w=8: \
        L.pww_sampler_update(eps, dt, 256, 1, 32, 4, lat, hist, hl, noise, gs, beta, form, m, h, w, None)  # noqa: E731
    for dt in (F16, BF16):
        for kw in ({"eps": None}, {"lat": None}, {"hist": None}, {"gs": None}, {"beta": None}, {"form": None},
                   {"m": 0}, {"h": 0}, {"w": 0}, {"hl": 0}, {"hl": 5}):
            assert upd(dt=dt, **kw) == -1, (dt, kw)
    assert upd(dt=2) == -2 and upd(dt=3) == -2 and upd(dt=5) == -2 and upd(dt=-1) == -2
    assert L.pww_status_str(-2).startswith(b"unsupported")


def test_dtype_codes():
    assert PL._dtype_code(torch.bfloat16) == _native.PWW_DTYPE_BF16 == 4
    assert PL._dtype_code(torch.float16) == 1 and PL._dtype_code(torch.float32) == 0
    assert PL._dtype_code(torch.float64) == -1


def test_load_tools_builds_a_bf16_unet_on_request():
    from paint_with_words_sd_b200 import attention
    try:
        _, unet, _, _, _ = PL.pww_load_tools("cpu", hf_model_path="synthetic:tiny", torch_dtype=torch.bfloat16)
        assert {p.dtype for p in unet.parameters()} == {torch.bfloat16}
        _, unet16, _, _, _ = PL.pww_load_tools("cpu", hf_model_path="synthetic:tiny", torch_dtype=None)
        assert {p.dtype for p in unet16.parameters()} == {torch.float16}
        # the same seeded weights, rounded to each type
        w32 = PL.pww_load_tools("cpu", hf_model_path="synthetic:tiny", torch_dtype=torch.float32)[1].conv_in.weight
        assert torch.equal(unet.conv_in.weight, w32.to(torch.bfloat16))
        assert torch.equal(unet16.conv_in.weight, w32.to(torch.float16))
    finally:
        attention.unpatch_all()


def test_public_functions_take_torch_dtype():
    import inspect
    for fn in (PL.paint_with_words, PL.paint_with_words_inpaint, PL.paint_with_words_batch, PL.pww_load_tools,
               PL.PaintWithWord_StableDiffusionPipeline.from_pretrained,
               PL.PaintWithWord_StableDiffusionInpaintPipeline.from_pretrained):
        assert inspect.signature(fn).parameters["torch_dtype"].default is None, fn
