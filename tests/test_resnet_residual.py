"""The ResNet residual epilogue's C entry points reject bad arguments before any CUDA call (no GPU needed)."""
import ctypes

import pytest

from paint_with_words_sd_b200 import _native


@pytest.mark.parametrize("name", ["pww_resnet_residual_f16", "pww_resnet_residual_bf16"])
def test_resnet_residual_rejects_bad_arguments(name):
    fn = getattr(_native.lib(), name)
    buf = (ctypes.c_char * 4096)()
    p = (ctypes.addressof(buf) + 15) // 16 * 16
    ok = dict(a=p, h=p + 1024, bias=p + 2048, out=p + 1024, rows=4, C=64)

    def call(**kw):
        a = {**ok, **kw}
        return fn(a["a"], a["h"], a["bias"], a["out"], a["rows"], a["C"], None)

    for ptr in ("a", "h", "bias", "out"):
        assert call(**{ptr: None}) == -1, f"null {ptr}"
        assert call(**{ptr: ok[ptr] + 2}) == -1, f"misaligned {ptr}"
    for bad in (dict(rows=0), dict(rows=-3), dict(C=0), dict(C=-8), dict(C=12), dict(C=4)):
        assert call(**bad) == -1, bad
