"""Python wrappers for the fused channels-last UNet ops of libpww_b200 (GroupNorm[+add][+SiLU], GEGLU, add+LayerNorm,
the ResNet residual epilogue, with or without a T2I-Adapter feature) and the ControlNet residual injection and
multi-ControlNet combine.

Used by `unet.py` on CUDA fp16 or bf16 activations (the `_f16` / `_bf16` entry points, picked from x.dtype); the
CPU/fp32 route of the same modules stays plain PyTorch (it is what the CPU reference arm runs).  No fallback on CUDA: a
non-zero status raises.
"""
from __future__ import annotations

import ctypes
from typing import Dict, Optional

import torch

from . import _native

_WS: Dict[torch.device, torch.Tensor] = {}


def _workspace(device, nbytes: int) -> torch.Tensor:
    """GroupNorm scratch.  A larger request gets a NEW buffer; the old one stays alive in `_WS_KEEP` because captured
    CUDA graphs may still hold its address (a graph only ever sees the buffer that was current when it was captured)."""
    w = _WS.get(device)
    if w is None or w.numel() < nbytes:
        if w is not None:
            _WS_KEEP.append(w)
        w = torch.empty(max(nbytes, 4 << 20), dtype=torch.uint8, device=device)
        _WS[device] = w
    return w


_WS_KEEP: list = []


ENABLED = True     # bench.py's eager-PyTorch comparison leg turns the fused UNet ops off (stock PyTorch route)


def is_fast(x: torch.Tensor) -> bool:
    return ENABLED and x.is_cuda and x.dtype in (torch.float16, torch.bfloat16)


def group_norm_nhwc(x: torch.Tensor, gn: torch.nn.GroupNorm, add: Optional[torch.Tensor] = None,
                    silu: bool = True) -> torch.Tensor:
    """x: [B,C,H,W] fp16 or bf16 in channels-last memory, gn's parameters of the same type.  Returns
    act(GroupNorm(x + add[:, :, None, None])), channels last; `add` is cast to x's type."""
    if not x.is_contiguous(memory_format=torch.channels_last):
        x = x.contiguous(memory_format=torch.channels_last)
    B, C, H, W = x.shape
    L = _native.lib()
    y = torch.empty_like(x, memory_format=torch.channels_last)
    nbytes = L.pww_groupnorm_workspace_bytes(B, H * W, gn.num_groups)
    ws = _workspace(x.device, nbytes)
    add_bs = 0
    if add is not None:
        if add.dtype != x.dtype or add.stride(-1) != 1 or (add.stride(0) % 8) or (add.data_ptr() % 16):
            add = add.to(x.dtype).contiguous()
        add_bs = add.stride(0)
    fn = _native.entry("pww_groupnorm_nhwc", x.dtype)
    with torch.cuda.device(x.device):
        rc = fn(x.data_ptr(), None if add is None else add.data_ptr(), add_bs, gn.weight.data_ptr(),
                gn.bias.data_ptr(), y.data_ptr(), B, H * W, C, gn.num_groups, float(gn.eps),
                1 if silu else 0, ws.data_ptr(), ws.numel(), torch.cuda.current_stream(x.device).cuda_stream)
    _native.check(rc, fn.__name__)
    _native.launch_count += 2
    return y


def geglu(h: torch.Tensor) -> torch.Tensor:
    """h: [..., 2*I] fp16 or bf16 contiguous -> [..., I] = h[..., :I] * gelu(h[..., I:])."""
    if not h.is_contiguous():
        h = h.contiguous()
    I = h.shape[-1] // 2
    M = h.numel() // h.shape[-1]
    out = torch.empty(h.shape[:-1] + (I,), dtype=h.dtype, device=h.device)
    fn = _native.entry("pww_geglu", h.dtype)
    with torch.cuda.device(h.device):
        rc = fn(h.data_ptr(), out.data_ptr(), M, I, torch.cuda.current_stream(h.device).cuda_stream)
    _native.check(rc, fn.__name__)
    _native.launch_count += 1
    return out


def add_layer_norm(x: torch.Tensor, res: Optional[torch.Tensor], ln: torch.nn.LayerNorm, want_sum: bool = True):
    """(s, y) with s = x + res (s is x itself when res is None) and y = LayerNorm(s); x, res: [..., C] fp16 or bf16
    (both of one type, ln's parameters too)."""
    if not x.is_contiguous():
        x = x.contiguous()
    if res is not None and not res.is_contiguous():
        res = res.contiguous()
    C = x.shape[-1]
    M = x.numel() // C
    y = torch.empty_like(x)
    s = torch.empty_like(x) if (res is not None and want_sum) else None
    fn = _native.entry("pww_add_layernorm", x.dtype)
    with torch.cuda.device(x.device):
        rc = fn(x.data_ptr(), None if res is None else res.data_ptr(), ln.weight.data_ptr(), ln.bias.data_ptr(),
                None if s is None else s.data_ptr(), y.data_ptr(), M, C, float(ln.eps),
                torch.cuda.current_stream(x.device).cuda_stream)
    _native.check(rc, fn.__name__)
    _native.launch_count += 1
    return (x if res is None else s), y


def resnet_residual(a: torch.Tensor, h: torch.Tensor, bias: torch.Tensor, out: Optional[torch.Tensor] = None):
    """out = (a.float() + h.float() + bias[None, :, None, None]).to(E) in one launch (`pww_resnet_residual_*`): a ResNet
    block's output from its identity or bias-free shortcut output `a` and its bias-free conv2 output `h`, both [B, C, H,
    W] of one type E (fp16 or bf16), made channels-last if they are not.  `bias`: fp32 [C] (conv2's bias plus the
    shortcut's).  `out` (channels-last) defaults to h (in place).  Returns out."""
    cl = torch.channels_last
    a, h = a.contiguous(memory_format=cl), h.contiguous(memory_format=cl)
    out = h if out is None else out
    C = h.shape[1]
    if (tuple(a.shape) != tuple(h.shape) or tuple(out.shape) != tuple(h.shape) or a.dtype != h.dtype
            or out.dtype != h.dtype or not all(t.is_contiguous(memory_format=cl) for t in (a, h, out))):
        raise ValueError(f"resnet_residual needs a, h and out of one shape and type, channels-last (got "
                         f"{tuple(a.shape)} {a.dtype}, {tuple(h.shape)} {h.dtype}, {tuple(out.shape)} {out.dtype})")
    if bias.dtype != torch.float32 or tuple(bias.shape) != (C,) or not bias.is_contiguous() or bias.device != h.device:
        raise ValueError(f"resnet_residual bias must be a contiguous fp32 [{C}] tensor on {h.device}")
    fn = _native.entry("pww_resnet_residual", h.dtype)
    with torch.cuda.device(h.device):
        rc = fn(a.data_ptr(), h.data_ptr(), bias.data_ptr(), out.data_ptr(), h.numel() // C, C,
                torch.cuda.current_stream(h.device).cuda_stream)
    _native.check(rc, fn.__name__)
    _native.launch_count += 1
    return out


def adapter_residual(a: torch.Tensor, b: torch.Tensor, bias: Optional[torch.Tensor], feat: Optional[torch.Tensor],
                     out: Optional[torch.Tensor] = None) -> torch.Tensor:
    """s = (a.float() + b.float() [+ bias]).to(E), then out[:r] = (s[:r].float() + feat.float()).to(E) and out[r:] =
    s[r:] (r = feat.shape[0], 0 for feat None), in one launch (`pww_adapter_residual_*`): a residual epilogue with a
    T2I-Adapter feature added before the skip is taken.  a, b: [rows, C, h, w] of one type E (fp16 or bf16), both
    channels-last; feat: [r <= rows, C, h, w] of that type and format; bias: fp32 [C] or None.  `out` (channels-last)
    defaults to b (in place).  Returns out."""
    cl = torch.channels_last
    out = b if out is None else out
    C = b.shape[1]
    ops = [("a", a), ("b", b), ("out", out)]
    for name, t in ops:
        if (t.dim() != 4 or tuple(t.shape) != tuple(b.shape) or t.dtype != b.dtype or t.device != b.device
                or not t.is_contiguous(memory_format=cl)):
            raise ValueError(f"adapter_residual {name} {tuple(t.shape)} {t.dtype} does not match b {tuple(b.shape)} "
                             f"{b.dtype} (a, b and out: one shape, type and device, channels-last)")
    rows = 0
    if feat is not None:
        rows = int(feat.shape[0]) if feat.dim() == 4 else -1
        if (feat.dim() != 4 or tuple(feat.shape[1:]) != tuple(b.shape[1:]) or rows > b.shape[0]
                or feat.dtype != b.dtype or feat.device != b.device or not feat.is_contiguous(memory_format=cl)):
            raise ValueError(f"adapter_residual feat {tuple(feat.shape)} {feat.dtype} does not match b "
                             f"{tuple(b.shape)} {b.dtype} (same type, channels and size, at most as many images, "
                             "channels-last)")
    if bias is not None and (bias.dtype != torch.float32 or tuple(bias.shape) != (C,) or not bias.is_contiguous()
                             or bias.device != b.device):
        raise ValueError(f"adapter_residual bias must be a contiguous fp32 [{C}] tensor on {b.device}")
    fn = _native.entry("pww_adapter_residual", b.dtype)
    with torch.cuda.device(b.device):
        rc = fn(a.data_ptr(), b.data_ptr(), None if bias is None else bias.data_ptr(),
                None if feat is None else feat.data_ptr(), out.data_ptr(), b.shape[0], b.shape[2] * b.shape[3], C,
                rows, torch.cuda.current_stream(b.device).cuda_stream)
    _native.check(rc, fn.__name__)
    _native.launch_count += 1
    return out


def _same_dense_layout(a: torch.Tensor, b: torch.Tensor) -> bool:
    """Both channels-last contiguous or both contiguous: element j of image i is at i * C*h*w + j in both."""
    cl = torch.channels_last
    return (a.is_contiguous(memory_format=cl) and b.is_contiguous(memory_format=cl)) or (a.is_contiguous()
                                                                                         and b.is_contiguous())


def control_inject(dst, res, scales: Optional[torch.Tensor] = None) -> None:
    """dst_k[:rows] += (res_k * scales[k, :, None, None, None]) in place for every k, in ONE launch
    (`pww_control_inject_*`); rows = res_k.shape[0] <= dst_k.shape[0], the product rounded to dst's type before the add.
    dst_k and res_k: [B, C, h, w] / [rows, C, h, w] of one element type and one memory format (channels-last in the
    UNet).  `scales`: fp32 [n, rows] on dst's device, or None for a scale of 1."""
    n = len(dst)
    if n != len(res) or n < 1:
        raise ValueError(f"control_inject needs as many residuals as targets (got {len(res)} for {n})")
    rows = int(res[0].shape[0])
    for k, (d, r) in enumerate(zip(dst, res)):
        if (tuple(r.shape[1:]) != tuple(d.shape[1:]) or r.shape[0] != rows or rows > d.shape[0] or r.dtype != d.dtype
                or r.device != d.device or not _same_dense_layout(d, r)):
            raise ValueError(f"residual {k} {tuple(r.shape)} {r.dtype} does not match its target {tuple(d.shape)} "
                             f"{d.dtype} (same type, format, channels and size, at most as many images)")
    if scales is not None and (scales.dtype != torch.float32 or tuple(scales.shape) != (n, rows)
                               or not scales.is_contiguous() or scales.device != dst[0].device):
        raise ValueError(f"control scales must be a contiguous fp32 [{n}, {rows}] tensor on {dst[0].device}")
    d0 = dst[0]
    fn = _native.entry("pww_control_inject", d0.dtype)
    ptrs = (ctypes.c_void_p * n)(*[d.data_ptr() for d in dst])
    rptrs = (ctypes.c_void_p * n)(*[r.data_ptr() for r in res])
    elems = (ctypes.c_int64 * n)(*[d[0].numel() for d in dst])
    with torch.cuda.device(d0.device):
        rc = fn(n, ptrs, rptrs, elems, rows, None if scales is None else scales.data_ptr(),
                torch.cuda.current_stream(d0.device).cuda_stream)
    _native.check(rc, fn.__name__)
    _native.launch_count += 1


def control_combine(res_per_unit, scales: torch.Tensor, out=None) -> list:
    """out_k = sum over units u, in order, of (res_per_unit[u][k] * scales[u, k, :, None, None, None]), each product and
    partial sum rounded to the residuals' type, for every level k in ONE launch (`pww_control_combine_*`).  Every
    unit gives n residuals [rows, C_k, h_k, w_k] of one element type and one memory format; `scales` is fp32
    [units, n, rows] on their device.  `out` (n tensors like unit 0's) defaults to unit 0's residuals: the sum goes
    in place.  Returns out."""
    units = len(res_per_unit)
    first = list(res_per_unit[0]) if units else []
    n = len(first)
    out = first if out is None else list(out)
    if units < 1 or n < 1 or len(out) != n or any(len(r) != n for r in res_per_unit):
        raise ValueError(f"control_combine needs n >= 1 residuals from each of >= 1 units and n outputs (got "
                         f"{[len(r) for r in res_per_unit]} residuals, {len(out)} outputs)")
    rows = int(first[0].shape[0])
    for k in range(n):
        ref = first[k]
        for u, r in enumerate([res_per_unit[u][k] for u in range(units)] + [out[k]]):
            if (tuple(r.shape) != tuple(ref.shape) or r.shape[0] != rows or r.dtype != ref.dtype
                    or r.device != ref.device or not _same_dense_layout(ref, r)):
                what = "output" if u == units else f"unit {u}'s residual"
                raise ValueError(f"{what} {k} {tuple(r.shape)} {r.dtype} does not match unit 0's {tuple(ref.shape)} "
                                 f"{ref.dtype} (same type, format, shape and device)")
    d0 = first[0]
    if (scales.dtype != torch.float32 or tuple(scales.shape) != (units, n, rows) or not scales.is_contiguous()
            or scales.device != d0.device):
        raise ValueError(f"control scales must be a contiguous fp32 [{units}, {n}, {rows}] tensor on {d0.device}")
    fn = _native.entry("pww_control_combine", d0.dtype)
    optrs = (ctypes.c_void_p * n)(*[o.data_ptr() for o in out])
    rptrs = (ctypes.c_void_p * (units * n))(*[r.data_ptr() for unit in res_per_unit for r in unit])
    elems = (ctypes.c_int64 * n)(*[r[0].numel() for r in first])
    with torch.cuda.device(d0.device):
        rc = fn(units, n, optrs, rptrs, elems, rows, scales.data_ptr(), torch.cuda.current_stream(d0.device).cuda_stream)
    _native.check(rc, fn.__name__)
    _native.launch_count += 1
    return out
