"""The drop-in boundary: `inj_forward`, the replacement for diffusers' `CrossAttention.__call__`.

Same calling convention, context-dict schema and patch mechanism as the reference
(paint_with_words/paint_with_words.py:60-125 `inj_forward`, 193-195 / 556-559 patch sites):

    inj_forward(self, hidden_states, context=None, mask=None) -> Tensor[B, N, C]
    context: None (self-attention) | Tensor[B,T,Dc] | dict with
        "CONTEXT_TENSOR", "CROSS_ATTENTION_WEIGHT_{N}" ([N,T] fp32 or int 0),
        "CROSS_ATTENTION_WEIGHT_ORIG" ([H,W,T] fp32 or int 0), "SIGMA", "WEIGHT_FUNCTION"
    T = 77 (one CLIP window, any T <= 80 works) or a long prompt of 2 or 3 concatenated 77-token chunks (T = 154, 231;
    `conditioning.chunk_prompt`, the A1111 / compel layout).
        (optional, ours) "WMAP_INDEX", "G_SIGMA", "STAT_KIND", "CROSS_ATTENTION_PACKED_{N}", "PWW_SCRATCH",
        "ATTN_RECORD" (per-region attention recording, see RECORD_KEY), "REGION_WEIGHTS_{N}" (region prompts: fp32
        [N, k] or [Bw, N, k] chunk weights of a k-chunk context, see cross_attention's `region`), "REGION_ROWS" and
        "REGION_STAT_CHUNKS" (negative region prompts: int32 [B] weight row and statistic chunks of every image, see
        cross_attention's `region_rows`)

Everything between the q/k/v projections and the output projection runs in libpww_b200.so through
the C ABI (include/pww_b200.h): ONE launch of `pww_xattn_fused_f16` (per-image max/std of QK^T over all heads,
bias from the packed weight map, softmax, PV).  Maps with more than 10 distinct columns take the dense pair
`pww_xattn_stats_f16` + `pww_xattn_fwd_f16`.  No score tensor, head permute or mask broadcast is materialised.
There is no PyTorch/CPU fallback for the cross-attention path: unsupported shapes or weight functions
raise.

Element type: a call runs in bf16 (the `_bf16` entry points) when q is bf16 and in fp16 otherwise; k and v are cast to
q's type and the output has it.  `inj_forward` runs the projections under a bf16 autocast when the module's weights are
bf16 and under an fp16 autocast otherwise, so a bf16 UNet keeps a bf16 residual stream.

Extensions beyond the reference (which is hard-wired to batch 1, paint_with_words.py:445):
  * B > 1 with per-image statistics -- each image's max/std is its own, so results do not depend on
    how images are batched or sharded across GPUs;
  * dict key "WMAP_INDEX" (int32 [B] device tensor): image b uses weight map `WMAP_INDEX[b]` of a
    stacked [Bw,N,77] map, -1 = no bias.  This is what lets the cond and uncond halves of
    classifier-free guidance run as ONE batch-2 forward instead of two (paint_with_words.py:483-499);
  * per-image weight functions: dict key "STAT_KIND" (int32 [B] device tensor, PWW_STAT_MAX / PWW_STAT_STD per image)
    with "G_SIGMA" holding B values, both kept by `PwWSampler`.  Image b's bias is G_SIGMA[b] * stat_b(qk) * w, and
    the call still is one launch (the `_multi` entry points).  A dict without "STAT_KIND" probes its one
    WEIGHT_FUNCTION as the reference does.
"""
from __future__ import annotations

import math
from typing import Dict, Optional, Union

import torch
import torch.nn.functional as F

from . import _native
from .conditioning import (PACK_TOKENS, REGION_ROWS_KEY, STAT_CHUNKS_KEY, expand_orig_weight_map, key_chunks,
                           pack_weight_map, packed_key, region_key, weight_key)
from .weight_function import g_of_sigma, probe_weight_function

_ORIG_KEY = "CROSS_ATTENTION_WEIGHT_ORIG"
# Attention recording (kept by PwWSampler(record_attention=True)): {N: (ridx, rec_index, rec_acc)}, the `record` of every
# cross-attention call with N query rows (see cross_attention).  A dict without it records nothing.
RECORD_KEY = "ATTN_RECORD"


class _DeviceState:
    """Per-device scratch owned by the shim: G(sigma) device scalar, stats [B], stats workspace."""

    def __init__(self, device: torch.device):
        self.device = device
        self.g_sigma = torch.zeros(1, dtype=torch.float32, device=device)
        self._g_key = None
        # Fixed-size scratch: captured CUDA graphs bake these addresses in, so they are never reallocated (ensure() raises
        # instead of growing them).  8 MiB of dense-path workspace covers 127 images per call.
        self.stats = torch.zeros(1024, dtype=torch.float32, device=device)
        self.workspace = torch.zeros(8 << 20, dtype=torch.uint8, device=device)
        # scratch of the one-launch kernel: fixed size, never reallocated (CUDA graphs bake its address in)
        self.fused_ws = torch.zeros(_native.lib().pww_xattn_fused_workspace_bytes(), dtype=torch.uint8, device=device)
        self.index_cache: Dict[int, torch.Tensor] = {}
        self.pack_cache: Dict[tuple, object] = {}

    def set_g(self, key, value: float) -> None:
        if key != self._g_key:
            self.g_sigma.fill_(value)      # async fill on the current stream; no host sync
            self._g_key = key

    def ensure(self, batch: int, ws_bytes: int) -> None:
        if self.stats.numel() < batch or self.workspace.numel() < ws_bytes:
            raise _native.NativeError(f"batch of {batch} images exceeds the shim's fixed scratch; split the call or pass "
                                      "your own stats_out/workspace")

    def packed(self, wmap: torch.Tensor):
        """Packed form of a dense device map, built once per (storage, version): the map is step-invariant, so the
        torch.unique + split below runs at the first call only (outside any graph capture).  The cache entry keeps a
        reference to the dense tensor: while it is cached its storage cannot be freed and handed to a different map with
        the same address, version and shape (which would make the key ambiguous)."""
        key = (wmap.data_ptr(), wmap._version, tuple(wmap.shape), tuple(wmap.stride()))
        hit = self.pack_cache.get(key)
        if hit is None:
            if torch.cuda.is_current_stream_capturing():
                raise _native.NativeError("weight map must be packed before CUDA-graph capture (run one eager step first "
                                          "or pass packed maps)")
            while len(self.pack_cache) >= 16:               # small FIFO: a sampler passes its own packed maps anyway
                self.pack_cache.pop(next(iter(self.pack_cache)))
            hit = (wmap, pack_weight_map(wmap) or False)
            self.pack_cache[key] = hit
        return hit[1] or None

    def shared_index(self, batch: int) -> torch.Tensor:
        t = self.index_cache.get(batch)
        if t is None:
            t = torch.zeros(batch, dtype=torch.int32, device=self.device)
            self.index_cache[batch] = t
        return t


_STATES: Dict[torch.device, _DeviceState] = {}


def _state(device: torch.device) -> _DeviceState:
    s = _STATES.get(device)
    if s is None:
        s = _STATES[device] = _DeviceState(device)
    return s


def reset_device_state() -> None:
    _STATES.clear()


def resolve_weight_map(context: dict, n: int, device):
    """`CROSS_ATTENTION_WEIGHT_{n}` lookup with the reference's ORIG fallback (paint_with_words.py:93-103),
    expanded once per n and cached in the dict instead of re-interpolated at every call."""
    try:
        return context[weight_key(n)]
    except KeyError:
        w = context[_ORIG_KEY]
        if isinstance(w, int):
            if context.get("ORIG_FALLBACK_DROPPED"):
                raise NotImplementedError(
                    f"no CROSS_ATTENTION_WEIGHT_{n} in a multi-image context: the ORIG-map fallback (paint_with_words.py:97-103) "
                    "is a single-image path; use sizes divisible by 64 or one image per sampler")
            return 0
        w = expand_orig_weight_map(w.detach().to("cpu", torch.float32), n).to(device)
        context[weight_key(n)] = w
        return w


def _elem_dtype(q: torch.Tensor) -> torch.dtype:
    """The element type the kernels run in for query q: bf16 for a bf16 q, fp16 for anything else."""
    return torch.bfloat16 if q.dtype == torch.bfloat16 else torch.float16


def _autocast_dtype(module) -> torch.dtype:
    """bf16 for a module with bf16 weights, fp16 otherwise (fp32 modules keep the reference's fp16 autocast)."""
    return torch.bfloat16 if module.to_q.weight.dtype == torch.bfloat16 else torch.float16


def _rows(t: torch.Tensor, dtype: torch.dtype = torch.float16) -> torch.Tensor:
    """[B,L,C] of `dtype` with unit channel stride and 16-byte friendly strides."""
    if t.dtype != dtype:
        t = t.to(dtype)
    if t.stride(-1) != 1 or (t.stride(0) % 8) or (t.stride(1) % 8) or (t.data_ptr() % 16):
        t = t.contiguous()
    return t


# "fused" / "auto" (default): ONE launch (statistic + bias + softmax + PV, packed maps; csrc/xattn_fused2.cuh) at every head
# dim -- it beats the two-launch pair at every SD1.5 and SD2.1 shape (cond + uncond launch, CUDA events, H100 80GB HBM3 at
# 700 W: N = 4096 d = 40: 26.9 vs 34.2 us; N = 1024 d = 80: 40.2 vs 48.4; N = 9216 d = 64: 40.2 vs 47.3); "dense": the
# pair of launches on the dense fp32 map, kept for maps that cannot be packed (> 10 distinct columns -- those always take
# it) and as a test / bench comparison.
XATTN_IMPL = "auto"


def cross_attention(q: torch.Tensor, k: torch.Tensor, v: torch.Tensor, heads: int, scale: float,
                    wmap: Optional[torch.Tensor] = None, wmap_index: Optional[torch.Tensor] = None,
                    stat: Union[int, torch.Tensor] = _native.PWW_STAT_MAX, g_sigma: Optional[torch.Tensor] = None,
                    return_stats: bool = False, packed=None, stats_out: Optional[torch.Tensor] = None,
                    workspace: Optional[torch.Tensor] = None, record=None, region: Optional[torch.Tensor] = None,
                    region_rows=None):
    """Fused region for a key sequence of T <= 80 tokens or of 2 / 3 CLIP chunks (T = 154, 231; any other T raises).
    q [B,N,C]; k,v [B,T,C]; wmap [Bw,N,T] fp32 or None; `packed` = (mpack [Bw,N,32] fp16, cidx [Bw,80 k] int8, k key
    chunks) from `conditioning.pack_weight_map` (built from `wmap` and cached when not given).  `stat` is one kind for
    every image (an int) with `g_sigma` a 1-element fp32 device tensor holding G(sigma), or per-image settings: an int32
    [B] device tensor of kinds with `g_sigma` an fp32 [B] device tensor (entry b = image b; the `_multi` entry points).
    `stats_out` / `workspace` let a caller that captures CUDA graphs own the scratch (defaults: per-device scratch of
    this module).  The call runs in bf16 when q is bf16 and in fp16 otherwise (see the module docstring).
    `record` = (ridx [Br, 80 k] int8, rec_index [B] int32, rec_acc [Br, heads, N, 16] fp32), all on q's device: the call
    goes to `pww_xattn_fused_rec_*`, which also adds every recorded image's per-region softmax mass into rec_acc
    (include/pww_b200.h).  It needs the one-launch kernel: a call that would take the dense pair raises.
    `region` = fp32 [Bw, N, k] chunk weights of a k = 2 or 3 chunk context (region prompts): the call goes to
    `pww_xattn_fused_region_*`, which gives every chunk its own softmax and mixes them per query row by these weights.
    Image b takes weight row `wmap_index[b]` (-1: (1, 0, ..), the first chunk alone), or row b without an index.  It
    needs the one-launch kernel and cannot record.
    `region_rows` = (region_index int32 [B], stat_chunks int32 [B] or None), on q's device, with `region`: image b
    takes weight row region_index[b] whether or not it is biased (wmap_index then only picks its map), and a biased
    image's statistic covers the chunks of its bit mask stat_chunks[b] (chunk 0 always; None: every chunk).  The call
    goes to `pww_xattn_fused_region_rows_*` (negative region prompts)."""
    L = _native.lib()
    dt = _elem_dtype(q)
    q, k, v = _rows(q, dt), _rows(k, dt), _rows(v, dt)
    B, N, C = q.shape
    T = k.shape[1]
    D = C // heads
    if k.stride() != v.stride():
        v = v.contiguous()
        k = k.contiguous()
    st = _state(q.device)
    with torch.cuda.device(q.device):               # native launches go to q's device whatever the current one is
        out = torch.empty((B, N, C), dtype=dt, device=q.device)
        stream = torch.cuda.current_stream(q.device).cuda_stream
        biased = wmap is not None or packed is not None
        if wmap is not None:
            if wmap.dim() == 2:
                wmap = wmap.unsqueeze(0)
            if wmap.shape[1] != N or wmap.shape[2] != T:
                raise ValueError(f"weight map shape {tuple(wmap.shape)} does not match N={N}, T={T}")
        impl = "dense" if XATTN_IMPL == "dense" else "fused"
        if impl == "dense" and biased and wmap is None:
            impl = "fused"                          # only the packed form was given
        if biased and packed is None and impl == "fused":
            if wmap.dtype != torch.float32 or not wmap.is_contiguous():
                wmap = wmap.to(torch.float32).contiguous()
            packed = st.packed(wmap)
        use_fused = impl == "fused" and (not biased or packed is not None)
        if biased and wmap_index is None:
            bw = packed[0].shape[0] if packed is not None else wmap.shape[0]
            wmap_index = st.shared_index(B) if bw == 1 else torch.arange(B, dtype=torch.int32, device=q.device)
        per_image = isinstance(stat, torch.Tensor)
        kind_ptr = None
        if per_image and biased:
            if (stat.dtype != torch.int32 or stat.numel() != B or not stat.is_contiguous() or stat.device != q.device
                    or g_sigma is None or g_sigma.dtype != torch.float32 or g_sigma.numel() != B
                    or not g_sigma.is_contiguous() or g_sigma.device != q.device):
                raise ValueError(f"per-image settings need an int32 [{B}] kind tensor and an fp32 [{B}] G tensor on "
                                 f"{q.device}")
            kind_ptr = stat.data_ptr()
        stats = None
        rec_args = ()
        region_args = ()
        if region is not None:
            kc = key_chunks(T)
            if region.dim() == 2:
                region = region.unsqueeze(0)
            if (kc < 2 or region.dtype != torch.float32 or region.dim() != 3 or tuple(region.shape[1:]) != (N, kc)
                    or not region[0].is_contiguous() or region.device != q.device):
                raise ValueError(f"region weights need fp32 [Bw, {N}, k] on {q.device} for a context of k = 2 or 3 "
                                 f"chunks (T = {T})")
            if not use_fused or record is not None:
                raise _native.NativeError("region prompts need the one-launch kernel without attention recording")
            if region_rows is not None:
                rows, chunks = region_rows
                for t in (rows,) if chunks is None else (rows, chunks):
                    if t.dtype != torch.int32 or t.numel() != B or not t.is_contiguous() or t.device != q.device:
                        raise ValueError(f"region_rows need int32 [{B}] region_index / stat_chunks on {q.device}")
                region_args = (region.data_ptr(), region.stride(0), rows.data_ptr(),
                               None if chunks is None else chunks.data_ptr())
            else:
                if wmap_index is None and region.shape[0] != B:
                    wmap_index = (st.shared_index(B) if region.shape[0] == 1 else None)
                    if wmap_index is None:
                        raise ValueError(f"{region.shape[0]} region weight rows for {B} images need a wmap_index")
                region_args = (region.data_ptr(), region.stride(0))
        if record is not None:
            if not use_fused:
                why = ("XATTN_IMPL is 'dense'" if impl == "dense" else
                       "the weight map has more than 10 distinct columns and takes the dense two-launch path")
                raise _native.NativeError(f"attention recording needs the one-launch kernel, but {why}")
            ridx, rec_index, rec_acc = record
            if (ridx.dtype != torch.int8 or ridx.dim() != 2 or ridx.shape[1] != PACK_TOKENS * max(1, key_chunks(T))
                    or not ridx.is_contiguous() or rec_index.dtype != torch.int32 or rec_index.numel() != B
                    or not rec_index.is_contiguous() or rec_acc.dtype != torch.float32 or rec_acc.dim() != 4
                    or tuple(rec_acc.shape[1:]) != (heads, N, 16) or not rec_acc[0].is_contiguous()
                    or any(t.device != q.device for t in (ridx, rec_index, rec_acc))):
                raise ValueError(f"record needs int8 [Br, {PACK_TOKENS * max(1, key_chunks(T))}] ridx, int32 [{B}] "
                                 f"rec_index and fp32 [Br, {heads}, {N}, 16] rec_acc on {q.device}")
            if not per_image and biased:           # the recording entry takes per-image kinds and G(sigma)
                stat = torch.full((B,), int(stat), dtype=torch.int32, device=q.device)
                g_sigma = g_sigma.reshape(-1)[:1].expand(B).contiguous()
                kind_ptr, per_image = stat.data_ptr(), True
            rec_args = (ridx.data_ptr(), rec_index.data_ptr(), rec_acc.data_ptr(), rec_acc.stride(0))
        if use_fused:
            mp_ptr = ci_ptr = idx_ptr = g_ptr = st_ptr = ws_ptr = None
            mp_bs = bw = ws_bytes = 0
            if biased:
                mpack, cidx = packed
                if (mpack.shape[1] != N or mpack.dtype != torch.float16 or cidx.dtype != torch.int8
                        or cidx.shape[-1] != PACK_TOKENS * max(1, key_chunks(T))):
                    raise ValueError("packed weight map does not match this attention level")
                st.ensure(B, 0)
                stats = st.stats if stats_out is None else stats_out
                ws = st.fused_ws if workspace is None else workspace
                mp_ptr, ci_ptr, idx_ptr = mpack.data_ptr(), cidx.data_ptr(), wmap_index.data_ptr()
                g_ptr, st_ptr, ws_ptr = g_sigma.data_ptr(), stats.data_ptr(), ws.data_ptr()
                mp_bs, bw, ws_bytes = mpack.stride(0), mpack.shape[0], ws.numel()
            if region_args and region_rows is None and wmap_index is not None:
                idx_ptr = wmap_index.data_ptr()    # the weight rows are reached through it with or without a bias
            name = "pww_xattn_fused_rec" if rec_args else ("pww_xattn_fused_multi" if per_image else "pww_xattn_fused")
            if region_args:
                name = "pww_xattn_fused_region_multi" if per_image else "pww_xattn_fused_region"
                if region_rows is not None:
                    name = name.replace("_region", "_region_rows")
            fn = _native.entry(name, dt)
            rc = fn(q.data_ptr(), k.data_ptr(), v.data_ptr(), out.data_ptr(), B, heads, N, T, D,
                    q.stride(0), q.stride(1), k.stride(0), k.stride(1), out.stride(0), out.stride(1),
                    mp_ptr, mp_bs, bw, ci_ptr, idx_ptr, kind_ptr if per_image or rec_args else stat, g_ptr,
                    float(scale), st_ptr, ws_ptr, ws_bytes, stream, *rec_args, *region_args)
            _native.check(rc, fn.__name__)
            _native.launch_count += 1
        else:
            stats_ptr = g_ptr = w_ptr = idx_ptr = None
            w_bs = 0
            if biased:
                if wmap is None:
                    raise ValueError("the dense path needs the dense weight map")
                if wmap.dtype != torch.float32 or not wmap.is_contiguous():
                    wmap = wmap.to(torch.float32).contiguous()
                ws_bytes = L.pww_xattn_workspace_bytes(B, heads, N, T, D)
                st.ensure(B, ws_bytes)
                stats = st.stats if stats_out is None else stats_out
                fn = _native.entry("pww_xattn_stats_multi" if per_image else "pww_xattn_stats", dt)
                rc = fn(q.data_ptr(), k.data_ptr(), B, heads, N, T, D, q.stride(0), q.stride(1), k.stride(0),
                        k.stride(1), kind_ptr if per_image else stat, wmap_index.data_ptr(), stats.data_ptr(),
                        st.workspace.data_ptr(), st.workspace.numel(), stream)
                _native.check(rc, fn.__name__)
                _native.launch_count += 1
                stats_ptr, g_ptr = stats.data_ptr(), g_sigma.data_ptr()
                w_ptr, idx_ptr, w_bs = wmap.data_ptr(), wmap_index.data_ptr(), wmap.stride(0)
            fn = _native.entry("pww_xattn_fwd_multi" if per_image else "pww_xattn_fwd", dt)
            rc = fn(q.data_ptr(), k.data_ptr(), v.data_ptr(), out.data_ptr(), B, heads, N, T, D,
                    q.stride(0), q.stride(1), k.stride(0), k.stride(1), out.stride(0), out.stride(1),
                    w_ptr, w_bs, idx_ptr, stats_ptr, g_ptr, float(scale), stream)
            _native.check(rc, fn.__name__)
            _native.launch_count += 1
    if return_stats:
        return out, (stats[:B].clone() if stats is not None else None)
    return out


# Self-attention (context=None): "native" = pww_attn_fwd_f16, the flash-attention kernel of libpww_b200 (csrc/attn_tc.cuh);
# "torch-sdpa" = torch's library attention -- like cuBLAS for the projections, a library call; "auto" (default) = whichever
# is faster on the H100: native up to 1024 keys, the library above.  Batch 2, CUDA events, H100 80GB HBM3 at 700 W, native
# vs library: N = 64 d = 160: 21 vs 29 us; N = 576 d = 64: 27 vs 42; N = 1024 d = 80: 33 vs 43; N = 256 d = 160: 31 vs 29;
# N = 2304 d = 64: 150 vs 71; N = 4096 d = 40: 284 vs 154.  bench.py records the setting in `config.self_attn`.
SELF_ATTN_IMPL = "auto"
SELF_ATTN_NATIVE_MAX_KEYS = 1024


def self_attention(q: torch.Tensor, k: torch.Tensor, v: torch.Tensor, heads: int, scale: float) -> torch.Tensor:
    B, N, C = q.shape
    D = C // heads
    if SELF_ATTN_IMPL == "native" or (SELF_ATTN_IMPL == "auto" and N <= SELF_ATTN_NATIVE_MAX_KEYS):
        dt = _elem_dtype(q)
        fn = _native.entry("pww_attn_fwd", dt)
        q, k, v = _rows(q, dt), _rows(k, dt), _rows(v, dt)
        if not (q.stride() == k.stride() == v.stride()):
            q, k, v = q.contiguous(), k.contiguous(), v.contiguous()
        with torch.cuda.device(q.device):
            out = torch.empty((B, N, C), dtype=dt, device=q.device)
            rc = fn(q.data_ptr(), k.data_ptr(), v.data_ptr(), out.data_ptr(), B, heads, N, D,
                    q.stride(0), q.stride(1), out.stride(0), out.stride(1), float(scale),
                    torch.cuda.current_stream(q.device).cuda_stream)
        _native.check(rc, fn.__name__)
        _native.launch_count += 1
        return out
    qh = q.reshape(B, N, heads, D).transpose(1, 2)
    kh = k.reshape(B, k.shape[1], heads, D).transpose(1, 2)
    vh = v.reshape(B, v.shape[1], heads, D).transpose(1, 2)
    o = F.scaled_dot_product_attention(qh, kh, vh, scale=scale)
    return o.transpose(1, 2).reshape(B, N, C)


def _fused_weight(module, attr: str, names) -> torch.Tensor:
    """Row-concatenated projection weights (to_q|to_k|to_v or to_k|to_v), built once per module: one GEMM instead of
    two or three.  The cache is keyed on the parameters' storage and version counters, so an in-place update of the
    weights (load_state_dict, a broadcast into the module after a first forward) rebuilds it."""
    params = [getattr(module, n).weight for n in names]
    key = tuple((p.data_ptr(), p._version, p.dtype, p.device) for p in params)
    hit = getattr(module, attr, None)
    if hit is None or hit[0] != key:
        hit = (key, torch.cat(params, 0).detach().contiguous())
        object.__setattr__(module, attr, hit)
    return hit[1]


def refresh_kv_cache(context: dict) -> None:
    """Recompute cached context K/V in place after CONTEXT_TENSOR changed (same storage: graph-replay safe)."""
    cache = context.get("KV_CACHE")
    if not cache:
        return
    ctx = context["CONTEXT_TENSOR"]
    for module, kv in cache.values():
        with torch.autocast("cuda", dtype=_autocast_dtype(module)):
            kv.copy_(F.linear(ctx, _fused_weight(module, "_pww_wkv", ("to_k", "to_v"))))


def inj_forward(self, hidden_states, context=None, mask=None):
    """Replacement for `CrossAttention.__call__` (reference: paint_with_words.py:60-125)."""
    if not hidden_states.is_cuda:
        raise _native.NativeError("paint_with_words_sd_b200 attention runs on an H100 GPU only (no CPU path)")
    is_dict = isinstance(context, dict)
    if context is None:
        ctx = hidden_states
    else:
        ctx = context["CONTEXT_TENSOR"] if is_dict else context

    C = self.to_q.weight.shape[0]
    act = _autocast_dtype(self)
    with torch.autocast("cuda", dtype=act):
        if context is None:
            # one [C -> 3C] GEMM; q/k/v are column views of its output (row stride 3C) -- the kernels take strides
            qkv = F.linear(hidden_states, _fused_weight(self, "_pww_wqkv", ("to_q", "to_k", "to_v")))
            q, k, v = qkv[..., :C], qkv[..., C:2 * C], qkv[..., 2 * C:]
        else:
            q = self.to_q(hidden_states)
            cache = context.get("KV_CACHE") if is_dict else None
            hit = cache.get(id(self)) if cache is not None else None
            if hit is not None:
                kv = hit[1]                          # K/V of the (step-invariant) text context, computed once
            else:
                kv = F.linear(ctx, _fused_weight(self, "_pww_wkv", ("to_k", "to_v")))
                if cache is not None:
                    cache[id(self)] = (self, kv)
            k, v = kv[..., :C], kv[..., C:]

    if context is None:
        o = self_attention(q, k, v, self.heads, self.scale)
    else:
        wmap = wmap_index = g_dev = packed = None
        scratch = (None, None)
        stat = _native.PWW_STAT_MAX
        kinds = context.get("STAT_KIND") if is_dict else None
        if kinds is not None:
            # per-image settings kept by PwWSampler: kinds [B] and G_SIGMA [B] on the device, WMAP_INDEX = -1 for the
            # images whose weight function is zero
            w = resolve_weight_map(context, q.shape[1], q.device)
            if isinstance(w, torch.Tensor):
                wmap, stat, g_dev = w, kinds, context["G_SIGMA"]
                wmap_index = context.get("WMAP_INDEX")
                packed = context.get(packed_key(q.shape[1]))
                scratch = context.get("PWW_SCRATCH", scratch)
        elif is_dict:
            f = context["WEIGHT_FUNCTION"]
            sigma = context["SIGMA"]
            w = resolve_weight_map(context, q.shape[1], q.device)
            probed = probe_weight_function(f, sigma)
            if isinstance(w, torch.Tensor) and not probed.is_zero:
                g_dev = context.get("G_SIGMA")      # device scalar kept by PwWSampler (graph replay safe)
                if g_dev is None:
                    st = _state(q.device)
                    st.set_g((id(f), float(sigma)), g_of_sigma(f, probed, sigma))
                    g_dev = st.g_sigma
                wmap, stat = w, probed.stat
                wmap_index = context.get("WMAP_INDEX")
                packed = context.get(packed_key(q.shape[1]))          # (mpack, cidx) prepared by PwWSampler
                scratch = context.get("PWW_SCRATCH", scratch)         # (stats, workspace) owned by the sampler
        record = None
        recs = context.get(RECORD_KEY) if is_dict else None
        if recs is not None:
            record = recs.get(q.shape[1])
            if record is None:
                raise _native.NativeError(f"attention recording has no accumulator for N = {q.shape[1]} query rows "
                                          f"(levels: {sorted(recs)})")
        region = context.get(region_key(q.shape[1])) if is_dict else None
        rows = context.get(REGION_ROWS_KEY) if region is not None else None
        if rows is not None:
            rows = (rows, context.get(STAT_CHUNKS_KEY))   # negative region prompts: weight rows of their own
        elif region is not None and wmap_index is None:
            wmap_index = context.get("WMAP_INDEX")      # the sampler's image -> weight row (-1: uncond images)
        if k.shape[0] != q.shape[0]:
            k = k.expand(q.shape[0], -1, -1)
            v = v.expand(q.shape[0], -1, -1)
        o = cross_attention(q, k, v, self.heads, self.scale, wmap, wmap_index, stat, g_dev, packed=packed,
                            stats_out=scratch[0], workspace=scratch[1], record=record, region=region,
                            region_rows=rows)

    with torch.autocast("cuda", dtype=act):
        o = self.to_out[0](o)
        o = self.to_out[1](o)
    return o


class PwWAttnProcessor:
    """diffusers>=0.12 `AttnProcessor`-style hook: `attn.set_processor(PwWAttnProcessor())`; the PwW context
    dict is passed as `encoder_hidden_states` exactly as with the class patch."""

    def __call__(self, attn, hidden_states, encoder_hidden_states=None, attention_mask=None, **kwargs):
        return inj_forward(attn, hidden_states, encoder_hidden_states, attention_mask)


_PATCHED: Dict[type, object] = {}


def patch_unet(unet, forward=inj_forward) -> int:
    """Class-level `__call__` patch of every module whose class is named "CrossAttention"
    (paint_with_words.py:193-195).  Returns the number of attention modules found."""
    count = 0
    for m in unet.modules():
        if m.__class__.__name__ == "CrossAttention":
            cls = m.__class__
            if cls not in _PATCHED:
                _PATCHED[cls] = cls.__dict__.get("__call__")
            cls.__call__ = forward
            count += 1
    return count


def unpatch_all() -> None:
    """Undo `patch_unet` (the reference never undoes its patch; tests need to)."""
    for cls, orig in _PATCHED.items():
        if orig is None:
            if "__call__" in cls.__dict__:
                delattr(cls, "__call__")
        else:
            cls.__call__ = orig
    _PATCHED.clear()
