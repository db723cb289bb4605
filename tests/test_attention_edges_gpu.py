"""Edge cases of the three attention kernels against one float64 reference: all-negative scores, a later key chunk that
dominates by tens of logits, broadcast (stride-0) contexts, inputs and outputs inside NaN-poisoned padded buffers, batch
splits of the one-launch ABI, the std statistic at full size and with a large mean, and short key lengths at every head
dim.

The reference (`_ref`) works per image in numpy float64 on the fp16 inputs: S = Q_h K_h^T per head; the statistic is the
max / std (ddof = 1) of fp16-rounded S over all heads, rows and tokens, rounded to fp16 (what the kernels and the
reference's autocast compute); the bias is g * stat * w; softmax and P.V in float64.  Tolerances are the suite's:
statistic |st - ref| <= 2^-10 |ref| + 1e-6, output max|got - ref| <= 2e-3 max|ref| per image, and bitwise equality where
two calls do the same computation by construction.
"""
import ctypes
import math

import numpy as np
import pytest
import torch

from oracle import pww_oracle as O
from paint_with_words_sd_b200 import _native
from paint_with_words_sd_b200 import attention as A
from paint_with_words_sd_b200.conditioning import pack_weight_map
from paint_with_words_sd_b200.unet import CrossAttention
from tests.test_xattn_gpu import IMPLS, _inputs, _run

pytestmark = pytest.mark.gpu

HEAD_DIMS = [(8, 40), (5, 64), (8, 80), (4, 160)]          # (heads, head dim)
G_MAX = 0.4 * math.log(1 + 7.0)
G_STD = 0.5 * math.log(1 + 7.0 ** 2)
NAN16 = 0x7E00                                             # fp16 quiet NaN: every gap element of an input buffer
SENTINEL = 0x7C01                                          # fp16 signalling NaN: every gap element of an output buffer


# ------------------------------------------------------------------------------------------------------------------
# float64 reference and checks
# ------------------------------------------------------------------------------------------------------------------
def _ref_image(q, k, v, H, scale, w, g, stat):
    """One image: q [N, C], k / v [T, C] (fp16 tensors), w [N, T] or None -> (out [N, C] float64, statistic)."""
    N, C = q.shape
    D = C // H
    qh = q.double().numpy().reshape(N, H, D).transpose(1, 0, 2)
    kh = k.double().numpy().reshape(-1, H, D).transpose(1, 0, 2)
    vh = v.double().numpy().reshape(-1, H, D).transpose(1, 0, 2)
    s = qh @ kh.transpose(0, 2, 1)                                   # [H, N, T], exact products of fp16 values
    st = 0.0
    if w is not None:
        s16 = s.astype(np.float16).astype(np.float64)
        st = float(np.float16(s16.max() if stat == "max" else s16.std(ddof=1)))
        s = s + g * st * np.asarray(w, dtype=np.float64)[None]
    s = s * scale
    s -= s.max(-1, keepdims=True)
    p = np.exp(s)
    p /= p.sum(-1, keepdims=True)
    return (p @ vh).transpose(1, 0, 2).reshape(N, C), st


def _ref(q, k, v, H, scale, maps, g, stat):
    """q [B, N, C], k / v [B, T, C]; maps[b] = image b's [N, T] weight map or None (no bias, statistic 0)."""
    outs, stats = [], []
    for b in range(q.shape[0]):
        o, st = _ref_image(q[b], k[b], v[b], H, scale, maps[b], g, stat)
        outs.append(o)
        stats.append(st)
    return np.stack(outs), stats


def _check(got, st, ref, ref_st, biased=None):
    """Per image: statistic within 2^-10 relative (exactly 0 for unbiased images); output within 2e-3 max|ref|."""
    got = np.asarray(got.float().cpu() if isinstance(got, torch.Tensor) else got, dtype=np.float64)
    for b in range(ref.shape[0]):
        if st is not None:
            s = float(st[b])
            if biased is not None and not biased[b]:
                assert s == 0.0, f"image {b}: unbiased image reports statistic {s}"
            else:
                assert abs(s - ref_st[b]) <= 2 ** -10 * abs(ref_st[b]) + 1e-6, f"image {b}: statistic {s} vs {ref_st[b]}"
        assert np.isfinite(got[b]).all(), f"image {b}: non-finite output"
        amax = np.abs(ref[b]).max()
        err = np.abs(got[b] - ref[b]).max()
        assert err <= 2e-3 * amax, f"image {b}: max|d| = {err:.3e} > 2e-3 * {amax:.3e}"


def _maps_for(w, idx):
    """Per-image maps of a stacked map `w` [Bw, N, T] under a map index (-1 = none)."""
    return [None if i < 0 else w[i].numpy() for i in idx]


def _shim(q, k, v, H, scale, w, g, stat, idx=None, impl="fused"):
    """`attention.cross_attention` on device tensors as given (their strides are kept)."""
    dev = q.device
    old = A.XATTN_IMPL
    A.XATTN_IMPL = impl
    try:
        out, st = A.cross_attention(q, k, v, H, scale, w, idx, _native.PWW_STAT_MAX if stat == "max" else _native.PWW_STAT_STD,
                                    torch.tensor([g], dtype=torch.float32, device=dev), return_stats=True)
        torch.cuda.synchronize()
    finally:
        A.XATTN_IMPL = old
    return out, st


def _sparse_maps(Bw, N, T, seed, cols=9):
    """Weight maps like the real ones: a few distinct non-zero columns per map (packable)."""
    g = torch.Generator().manual_seed(seed)
    w = torch.zeros(Bw, N, T)
    for b in range(Bw):
        for c in torch.randperm(T, generator=g)[:cols]:
            w[b, :, c] = (torch.rand(N, generator=g) > 0.5).float() * float(0.2 + torch.rand(1, generator=g) * 1.8)
    return w


# ------------------------------------------------------------------------------------------------------------------
# A. negative-score maxima: a padded score is exactly 0, so a leaking row or token mask makes the maximum read 0
# ------------------------------------------------------------------------------------------------------------------
def _negative(B, N, H, D, T, seed):
    q, k, v, w = _inputs(B, N, H, D, T, seed)
    return q.abs(), -k.abs(), v, w                        # every product q_d k_d <= 0: every score is strictly negative


@pytest.mark.parametrize("impl", IMPLS)
@pytest.mark.parametrize("T", [16, 41, 77, 154, 231])
@pytest.mark.parametrize("H,D", HEAD_DIMS)
@pytest.mark.parametrize("N", [1, 100, 129, 333, 1024])
def test_negative_scores_max(N, H, D, T, impl):
    q, k, v, w = _negative(1, N, H, D, T, seed=N * 7 + D + T)
    scale = D ** -0.5
    ref, ref_st = _ref(q, k, v, H, scale, [w[0].numpy()], G_MAX, "max")
    assert ref_st[0] < 0.0
    got, st = _run(q, k, v, H, scale, w, G_MAX, "max", impl=impl)
    _check(got, st, ref, ref_st)


@pytest.mark.parametrize("impl", IMPLS)
@pytest.mark.parametrize("T", [77, 231])
def test_negative_scores_batched_with_uncond_and_positive_image(T, impl):
    """[negative image, uncond, positive image] in one call: each image's maximum is its own."""
    N, H, D = 333, 8, 40
    q, k, v, _ = _inputs(3, N, H, D, T, seed=123 + T)
    q[0], k[0] = q[0].abs(), -k[0].abs()
    w = _sparse_maps(2, N, T, seed=T)
    idx = [1, -1, 0]
    ref, ref_st = _ref(q, k, v, H, D ** -0.5, _maps_for(w, idx), G_MAX, "max")
    assert ref_st[0] < 0.0 < ref_st[2]
    got, st = _run(q, k, v, H, D ** -0.5, w, G_MAX, "max", torch.tensor(idx, dtype=torch.int32), impl=impl)
    _check(got, st, ref, ref_st, biased=[i >= 0 for i in idx])


# ------------------------------------------------------------------------------------------------------------------
# B. streaming softmax over key chunks when the row maximum moves by tens of logits
# ------------------------------------------------------------------------------------------------------------------
def _chunk_dominance(N, H, D, T, dominant, seed, rise=48.0):
    """Q and the keys of chunk `dominant` share a per-head direction u_h: that chunk's scores sit ~`rise` logits above the
    others', so the running maximum jumps when it arrives (last chunk) or the later chunks underflow (first chunk)."""
    q, k, v, _ = _inputs(1, N, H, D, T, seed)
    g = torch.Generator().manual_seed(seed + 1)
    u = torch.randn(H, D, generator=g)
    u = u / u.norm(dim=1, keepdim=True)
    a = math.sqrt(rise / D ** -0.5)
    q = (q.float() + a * u.reshape(1, 1, H * D)).half()
    c = dominant * 77
    k[:, c:c + 77] = (k[:, c:c + 77].float() + a * u.reshape(1, 1, H * D)).half()
    return q, k, v


def _chunk_gap(q, k, H, scale, dominant):
    """Per row and head: (max over the dominant chunk) - (max over the other chunks), in logits."""
    N, C = q.shape[1:]
    D = C // H
    qh = q[0].double().numpy().reshape(N, H, D).transpose(1, 0, 2)
    kh = k[0].double().numpy().reshape(-1, H, D).transpose(1, 0, 2)
    s = (qh @ kh.transpose(0, 2, 1)) * scale
    inside = np.zeros(s.shape[-1], dtype=bool)
    inside[dominant * 77:dominant * 77 + 77] = True
    return s[..., inside].max(-1) - s[..., ~inside].max(-1)


@pytest.mark.parametrize("impl", IMPLS)
@pytest.mark.parametrize("stat", ["max", "std"])
@pytest.mark.parametrize("where", ["last", "first"])
@pytest.mark.parametrize("T", [154, 231])
@pytest.mark.parametrize("N,H,D", [(333, 8, 40), (256, 5, 64), (333, 4, 80), (129, 2, 160)])
def test_dominant_chunk(N, H, D, T, where, stat, impl):
    """Head dim 80 at 3 chunks and 160 at 2 and 3 run on one operand stage; every head dim is covered."""
    dom = T // 77 - 1 if where == "last" else 0
    q, k, v = _chunk_dominance(N, H, D, T, dom, seed=N + D + T)
    scale = D ** -0.5
    assert _chunk_gap(q, k, H, scale, dom).min() >= 30.0            # every row's maximum moves by >= 30 logits
    w = _sparse_maps(1, N, T, seed=D + T)
    g = 0.05                                                          # a bias of a few logits, not enough to mask the jump
    ref, ref_st = _ref(q, k, v, H, scale, [w[0].numpy()], g, stat)
    got, st = _run(q, k, v, H, scale, w, g, stat, impl=impl)
    _check(got, st, ref, ref_st)


@pytest.mark.parametrize("impl", IMPLS)
@pytest.mark.parametrize("stat", ["max", "std"])
@pytest.mark.parametrize("H,D", HEAD_DIMS)
def test_large_bias_in_the_third_chunk(H, D, stat, impl):
    """Strength-8 regions with g = 3 on tokens >= 154 only: biased logits of several hundred appear in the last chunk
    (the hi/lo map precision case of the single-chunk suite, moved behind two chunks of the streaming softmax)."""
    N, T = 333, 231
    q, k, v, _ = _inputs(1, N, H, D, T, seed=41 + D)
    gen = torch.Generator().manual_seed(9)
    base = torch.rand(N, 3, generator=gen) * 8.0
    w = torch.zeros(1, N, T)
    w[0, :, 158] = base[:, 0]; w[0, :, 159] = base[:, 0]; w[0, :, 174] = base[:, 1] + base[:, 0]; w[0, :, 187] = base[:, 2]
    ref, ref_st = _ref(q, k, v, H, D ** -0.5, [w[0].numpy()], 3.0, stat)
    got, st = _run(q, k, v, H, D ** -0.5, w, 3.0, stat, impl=impl)
    _check(got, st, ref, ref_st)


# ------------------------------------------------------------------------------------------------------------------
# C. a batch-1 context broadcast over the batch (k / v batch stride 0)
# ------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("impl", IMPLS)
@pytest.mark.parametrize("biased", [True, False])
@pytest.mark.parametrize("T", [77, 154])
@pytest.mark.parametrize("B", [2, 3])
def test_broadcast_context_is_bitwise_equal_to_copies(B, T, biased, impl):
    N, H, D = 333, 8, 40
    q, k, v, _ = _inputs(B, N, H, D, T, seed=B * 10 + T)
    w = _sparse_maps(B, N, T, seed=B + T) if biased else None
    idx = ([0, -1, 1][:B] if B == 3 else [0, -1]) if biased else None
    qd, k1, v1 = q.cuda(), k[:1].cuda(), v[:1].cuda()
    kx, vx = k1.expand(B, -1, -1), v1.expand(B, -1, -1)
    assert kx.stride(0) == 0 and A._rows(kx).stride(0) == 0          # the kernels get k_batch_stride = 0
    idx_d = None if idx is None else torch.tensor(idx, dtype=torch.int32, device="cuda")
    wd = None if w is None else w.cuda()
    got, st = _shim(qd, kx, vx, H, D ** -0.5, wd, G_MAX, "max", idx_d, impl)
    copy, st_copy = _shim(qd, kx.contiguous(), vx.contiguous(), H, D ** -0.5, wd, G_MAX, "max", idx_d, impl)
    assert torch.equal(got, copy)
    assert (st is None and st_copy is None) or torch.equal(st, st_copy)
    kb, vb = k[:1].expand(B, -1, -1), v[:1].expand(B, -1, -1)
    maps = _maps_for(w, idx) if biased else [None] * B
    ref, ref_st = _ref(q, kb, vb, H, D ** -0.5, maps, G_MAX, "max")
    _check(got, st, ref, ref_st, biased=[m is not None for m in maps])


@torch.no_grad()
def test_inj_forward_broadcasts_a_batch1_context():
    """inj_forward with batch-2 hidden states and a batch-1 context (dict with a weight map, and a plain tensor): the
    reference restatement is given the context expanded to batch 2.  Projection weights of 1.5 / sqrt(fan_in) spread the
    logits over ~2 units: much peakier scores would make the fp16 rounding of q, k and the statistic alone (the fp32 and
    the fp16-emulating oracle differ by 2e-3 max|out| at a 13-logit spread) use up the tolerance."""
    g = torch.Generator().manual_seed(17)
    heads, d, N, dc, T = 8, 40, 256, 64, 77
    attn = CrossAttention(heads * d, dc, heads, d)
    for p in attn.parameters():
        p.data = torch.randn(p.shape, generator=g) * (1.5 / math.sqrt(p.shape[1]) if p.dim() > 1 else 0.05)
    attn_d = CrossAttention(heads * d, dc, heads, d).cuda()
    attn_d.load_state_dict(attn.state_dict())
    x = torch.randn(2, N, heads * d, generator=g)
    ctx = torch.randn(1, T, dc, generator=g)
    w = _sparse_maps(1, N, T, seed=3)[0]
    f = lambda w_, sigma, qk: 0.4 * w_ * math.log(1 + sigma) * qk.max()   # noqa: E731
    sigma = torch.tensor(7.25)
    c = {f"CROSS_ATTENTION_WEIGHT_{N}": w, "CROSS_ATTENTION_WEIGHT_ORIG": 0, "SIGMA": sigma, "WEIGHT_FUNCTION": f}
    ref = O.inj_forward(attn, x, dict(c, CONTEXT_TENSOR=ctx.expand(2, -1, -1)))
    cd = dict(c, CONTEXT_TENSOR=ctx.cuda())
    cd[f"CROSS_ATTENTION_WEIGHT_{N}"] = w.cuda()
    got = A.inj_forward(attn_d, x.cuda(), cd).float().cpu()
    assert (got - ref).abs().max().item() <= 2e-3 * ref.abs().max().item()
    ref = O.inj_forward(attn, x, ctx.expand(2, -1, -1))
    got = A.inj_forward(attn_d, x.cuda(), ctx.cuda()).float().cpu()
    assert (got - ref).abs().max().item() <= 2e-3 * ref.abs().max().item()


# ------------------------------------------------------------------------------------------------------------------
# D. padded row / batch strides with NaN in every gap, through the C ABI
# ------------------------------------------------------------------------------------------------------------------
PAD_COLS, PAD_ROWS = 24, 3


def _poisoned(x, fill=NAN16):
    """x [B, L, C] inside a buffer [B, L + 3, C + 24] whose other elements hold the bit pattern `fill`; returns (buffer,
    view): row stride C + 24, batch stride (L + 3)(C + 24)."""
    B, L, C = x.shape
    buf = torch.empty(B, L + PAD_ROWS, C + PAD_COLS, dtype=torch.float16, device="cuda")
    buf.view(torch.int16).fill_(fill)
    view = buf[:, :L, :C]
    view.copy_(x)
    return buf, view


def _dense(x):
    """x as a contiguous device tensor followed by 256 spare elements, so that no read just past its end can leave the
    allocation whatever the kernel does."""
    flat = torch.zeros(x.numel() + 256, dtype=torch.float16, device="cuda")
    t = flat[:x.numel()].view(x.shape)
    t.copy_(x)
    return t


def _sentinel_out(B, L, C):
    """An output view [B, L, C] padded like `_poisoned`, every element of the buffer set to the sentinel."""
    buf = torch.empty(B, L + PAD_ROWS, C + PAD_COLS, dtype=torch.float16, device="cuda")
    buf.view(torch.int16).fill_(SENTINEL)
    return buf, buf[:, :L, :C]


def _gap_intact(buf, L, C):
    gap = torch.ones(buf.shape, dtype=torch.bool, device=buf.device)
    gap[:, :L, :C] = False
    return bool((buf.view(torch.int16)[gap] == SENTINEL).all())


def _stream():
    return torch.cuda.current_stream().cuda_stream


def _abi_fused(q, k, v, out, H, T, scale, packed=None, idx=None, stat="max", g=0.0, stats=None):
    """pww_xattn_fused_f16 on the given views; packed = (mpack, cidx) or None (plain); idx = None: identity mapping."""
    L = _native.lib()
    B, N, C = q.shape
    D = C // H
    mp = ci = ip = gp = sp = ws = None
    mp_bs = bw = ws_bytes = 0
    keep = []
    if packed is not None:
        mpack, cidx = packed
        gt = torch.tensor([g], dtype=torch.float32, device="cuda")
        wst = torch.zeros(L.pww_xattn_fused_workspace_bytes(), dtype=torch.uint8, device="cuda")
        keep += [gt, wst]
        mp, ci, gp, ws = mpack.data_ptr(), cidx.data_ptr(), gt.data_ptr(), wst.data_ptr()
        mp_bs, bw, ws_bytes = mpack.stride(0), mpack.shape[0], wst.numel()
        ip = None if idx is None else idx.data_ptr()
        sp = stats.data_ptr()
    rc = L.pww_xattn_fused_f16(q.data_ptr(), k.data_ptr(), v.data_ptr(), out.data_ptr(), B, H, N, T, D,
                               q.stride(0), q.stride(1), k.stride(0), k.stride(1), out.stride(0), out.stride(1),
                               mp, mp_bs, bw, ci, ip, 0 if stat == "max" else 1, gp, float(scale), sp, ws, ws_bytes,
                               _stream())
    _native.check(rc, "pww_xattn_fused_f16")
    torch.cuda.synchronize()


def _abi_dense(q, k, v, out, H, T, scale, wmap, idx, stat, g, stats):
    """pww_xattn_stats_f16 + pww_xattn_fwd_f16 on the given views, dense fp32 maps."""
    L = _native.lib()
    B, N, C = q.shape
    D = C // H
    ws = torch.zeros(L.pww_xattn_workspace_bytes(B, H, N, T, D), dtype=torch.uint8, device="cuda")
    gt = torch.tensor([g], dtype=torch.float32, device="cuda")
    st = 0 if stat == "max" else 1
    rc = L.pww_xattn_stats_f16(q.data_ptr(), k.data_ptr(), B, H, N, T, D, q.stride(0), q.stride(1), k.stride(0),
                               k.stride(1), st, idx.data_ptr(), stats.data_ptr(), ws.data_ptr(), ws.numel(), _stream())
    _native.check(rc, "pww_xattn_stats_f16")
    rc = L.pww_xattn_fwd_f16(q.data_ptr(), k.data_ptr(), v.data_ptr(), out.data_ptr(), B, H, N, T, D, q.stride(0),
                             q.stride(1), k.stride(0), k.stride(1), out.stride(0), out.stride(1), wmap.data_ptr(),
                             wmap.stride(0), idx.data_ptr(), stats.data_ptr(), gt.data_ptr(), float(scale), _stream())
    _native.check(rc, "pww_xattn_fwd_f16")
    torch.cuda.synchronize()


POISON_SHAPES = [(129, 8, 40), (129, 2, 160)]      # head dim 40: the last head's padding columns (40..47) are in the gap


def _poison_case(N, H, D, T, seed):
    """Two images: (host q, k, v), their poisoned views with a sentinel-filled padded output, and contiguous copies."""
    q, k, v, _ = _inputs(2, N, H, D, T, seed)
    C = H * D
    (_, qv), (_, kv), (_, vv) = _poisoned(q), _poisoned(k), _poisoned(v)
    ob, ov = _sentinel_out(2, N, C)
    assert kv.stride() == vv.stride() and qv.stride(1) == C + PAD_COLS
    dense = [_dense(t) for t in (q, k, v, torch.zeros(2, N, C))]
    return (q, k, v), (qv, kv, vv, ob, ov), dense


@pytest.mark.parametrize("mapped", [True, False])
@pytest.mark.parametrize("T", [77, 154])
@pytest.mark.parametrize("N,H,D", POISON_SHAPES)
def test_poisoned_views_fused(N, H, D, T, mapped):
    (q, k, v), (qv, kv, vv, ob, ov), (qc, kc, vc, oc) = _poison_case(N, H, D, T, seed=N + D + T)
    scale = D ** -0.5
    idx_l = [0, -1]
    packed = idx = None
    stats = torch.full((2,), -1.0, device="cuda")
    stats_c = stats.clone()
    w = _sparse_maps(1, N, T, seed=T)
    if mapped:
        packed = pack_weight_map(w.cuda())
        idx = torch.tensor(idx_l, dtype=torch.int32, device="cuda")
    _abi_fused(qv, kv, vv, ov, H, T, scale, packed, idx, "max", G_MAX, stats)
    _abi_fused(qc, kc, vc, oc, H, T, scale, packed, idx, "max", G_MAX, stats_c)
    assert torch.isfinite(ov).all()
    assert torch.equal(ov.view(torch.int16), oc.view(torch.int16))
    assert _gap_intact(ob, N, H * D)
    maps = _maps_for(w, idx_l) if mapped else [None, None]
    ref, ref_st = _ref(q, k, v, H, scale, maps, G_MAX, "max")
    _check(ov, stats.cpu() if mapped else None, ref, ref_st, biased=[m is not None for m in maps])
    if mapped:
        assert torch.equal(stats, stats_c)


@pytest.mark.parametrize("stat", ["max", "std"])
@pytest.mark.parametrize("T", [77, 154])
@pytest.mark.parametrize("N,H,D", POISON_SHAPES)
def test_poisoned_views_dense_pair(N, H, D, T, stat):
    (q, k, v), (qv, kv, vv, ob, ov), (qc, kc, vc, oc) = _poison_case(N, H, D, T, seed=N + D + T + 1)
    scale = D ** -0.5
    g = G_MAX if stat == "max" else G_STD
    w = _sparse_maps(1, N, T, seed=T + 1)
    wd = w.cuda()
    idx_l = [-1, 0]
    idx = torch.tensor(idx_l, dtype=torch.int32, device="cuda")
    stats = torch.full((2,), -1.0, device="cuda")
    stats_c = stats.clone()
    _abi_dense(qv, kv, vv, ov, H, T, scale, wd, idx, stat, g, stats)
    _abi_dense(qc, kc, vc, oc, H, T, scale, wd, idx, stat, g, stats_c)
    assert torch.isfinite(ov).all()
    assert torch.equal(ov.view(torch.int16), oc.view(torch.int16)) and torch.equal(stats, stats_c)
    assert _gap_intact(ob, N, H * D)
    ref, ref_st = _ref(q, k, v, H, scale, _maps_for(w, idx_l), g, stat)
    _check(ov, stats.cpu(), ref, ref_st, biased=[i >= 0 for i in idx_l])


@pytest.mark.parametrize("N,H,D", POISON_SHAPES)
def test_poisoned_views_self_attention(N, H, D):
    (q, k, v), (qv, kv, vv, ob, ov), (qc, kc, vc, oc) = _poison_case(N, H, D, N, seed=N + D + 2)   # N keys
    L = _native.lib()
    scale = D ** -0.5
    for (a, b_, c, o) in ((qv, kv, vv, ov), (qc, kc, vc, oc)):
        assert a.stride() == b_.stride() == c.stride()
        rc = L.pww_attn_fwd_f16(a.data_ptr(), b_.data_ptr(), c.data_ptr(), o.data_ptr(), 2, H, N, D, a.stride(0),
                                a.stride(1), o.stride(0), o.stride(1), float(scale), _stream())
        _native.check(rc, "pww_attn_fwd_f16")
    torch.cuda.synchronize()
    assert torch.isfinite(ov).all()
    assert torch.equal(ov.view(torch.int16), oc.view(torch.int16))
    assert _gap_intact(ob, N, H * D)
    ref, _ = _ref(q, k, v, H, scale, [None, None], 0.0, "max")
    _check(ov, None, ref, None)


# ------------------------------------------------------------------------------------------------------------------
# E. batches the one-launch ABI splits (more than 32 images, or a launch that does not fit and is halved)
# ------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("stat", ["max", "std"])
@pytest.mark.parametrize("N,H,D", [(129, 8, 40), (64, 4, 160)])
@pytest.mark.parametrize("B", [33, 40])
def test_fused_batch_split_with_map_index(B, N, H, D, stat):
    """More than 32 images: the second launch's images use maps from anywhere in a 48-map stack (indices above 31)."""
    T, Bw = 77, 48
    q, k, v, _ = _inputs(B, N, H, D, T, seed=B + D)
    w = _sparse_maps(Bw, N, T, seed=B)
    idx = [-1 if b % 4 == 1 else (7 * b + 5) % Bw for b in range(B)]
    assert idx[32] > 31 and -1 in idx[:32] and any(i > 31 for i in idx[:32])
    g = G_MAX if stat == "max" else G_STD
    got, st = _run(q, k, v, H, D ** -0.5, w, g, stat, torch.tensor(idx, dtype=torch.int32), impl="fused")
    ref, ref_st = _ref(q, k, v, H, D ** -0.5, _maps_for(w, idx), g, stat)
    _check(got, st, ref, ref_st, biased=[i >= 0 for i in idx])
    if stat == "max":                                   # batching does not change an image's result
        for b in range(B):
            wb = None if idx[b] < 0 else w[idx[b]:idx[b] + 1].contiguous()
            solo, _ = _run(q[b:b + 1], k[b:b + 1], v[b:b + 1], H, D ** -0.5, wb, g, stat, impl="fused")
            assert torch.equal(solo[0], got[b]), f"image {b}"


def _identity_call(q, k, v, H, w, g, stat):
    """pww_xattn_fused_f16 with wmap_index = NULL (image b uses map b), Bw = B, on contiguous device tensors."""
    B, N, C = q.shape
    qd, kd, vd = _dense(q), _dense(k), _dense(v)
    out = _dense(torch.zeros(B, N, C))
    stats = torch.full((B,), -1.0, device="cuda")
    _abi_fused(qd, kd, vd, out, H, k.shape[1], (C // H) ** -0.5, pack_weight_map(w.cuda()), None, stat, g, stats)
    return out, stats


@pytest.mark.parametrize("stat", ["max", "std"])
@pytest.mark.parametrize("T", [77, 231])
@pytest.mark.parametrize("B", [33, 40])
def test_fused_batch_split_identity_mapping(B, T, stat):
    """wmap_index = NULL across the split: the second launch's packed maps and column indices start at map 32."""
    N, H, D = 129, 8, 40
    q, k, v, _ = _inputs(B, N, H, D, T, seed=B + T)
    w = _sparse_maps(B, N, T, seed=B * T)
    g = G_MAX if stat == "max" else G_STD
    out, stats = _identity_call(q, k, v, H, w, g, stat)
    ref, ref_st = _ref(q, k, v, H, D ** -0.5, [w[b].numpy() for b in range(B)], g, stat)
    _check(out, stats.cpu(), ref, ref_st)
    # the same call with an explicit 0..B-1 index does the same work
    got, st = _run(q, k, v, H, D ** -0.5, w, g, stat, torch.arange(B, dtype=torch.int32), impl="fused")
    assert torch.equal(out.float().cpu(), got) and torch.equal(stats.cpu(), st)


def _set_fused_grid(n):
    L = _native.lib()
    L.pww_debug_set_fused_grid.argtypes = [ctypes.c_int]
    assert L.pww_debug_set_fused_grid(n) == 0


@pytest.mark.parametrize("stat", ["max", "std"])
def test_fused_forced_halving(stat):
    """A 2-CTA grid cannot hold 32 images of (N 1024, 8 heads of 40): the ABI halves the images per launch down to 2
    (16 launches), with identity-mapped maps offset at every launch."""
    B, N, H, D, T = 32, 1024, 8, 40, 77
    q, k, v, _ = _inputs(B, N, H, D, T, seed=2024)
    w = _sparse_maps(B, N, T, seed=11)
    g = G_MAX if stat == "max" else G_STD
    L = _native.lib()
    dump = torch.zeros(2 * (2 + 1024), dtype=torch.int32, device="cuda")
    L.pww_debug_set_fused_jobs_dump.argtypes = [ctypes.c_void_p]
    _set_fused_grid(2)
    L.pww_debug_set_fused_jobs_dump(dump.data_ptr())
    try:
        out, stats = _identity_call(q, k, v, H, w, g, stat)
    finally:
        L.pww_debug_set_fused_jobs_dump(None)
        _set_fused_grid(0)
    d = dump.cpu().numpy().reshape(2, 2 + 1024)
    # the last launch: 2 images x 4 head groups x 8 row tiles = 64 units, 32 per CTA -> 64 statistic + 64 softmax jobs
    assert d[:, 0].tolist() == [128, 128] and d[:, 1].tolist() == [64, 64]
    ref, ref_st = _ref(q, k, v, H, D ** -0.5, [w[b].numpy() for b in range(B)], g, stat)
    _check(out, stats.cpu(), ref, ref_st)
    if stat == "max":                                   # the statistic does not depend on the split or the grid
        full, st_full = _identity_call(q, k, v, H, w, g, stat)
        assert torch.equal(full.view(torch.int16), out.view(torch.int16)) and torch.equal(st_full, stats)


@pytest.mark.parametrize("stat", ["max", "std"])
def test_dense_pair_large_batch_through_the_shim(stat):
    """100 images (50 cond + 50 uncond) in one call of the dense pair: the shim's fixed workspace covers 127."""
    B, N, H, D, T = 100, 64, 8, 160, 77
    q, k, v, _ = _inputs(B, N, H, D, T, seed=100)
    w = _sparse_maps(B // 2, N, T, seed=50)
    idx = [b // 2 if b % 2 == 0 else -1 for b in range(B)]
    g = G_MAX if stat == "max" else G_STD
    got, st = _run(q, k, v, H, D ** -0.5, w, g, stat, torch.tensor(idx, dtype=torch.int32), impl="dense")
    ref, ref_st = _ref(q, k, v, H, D ** -0.5, _maps_for(w, idx), g, stat)
    _check(got, st, ref, ref_st, biased=[i >= 0 for i in idx])
    if stat == "max":
        for b in range(B):
            wb = None if idx[b] < 0 else w[idx[b]:idx[b] + 1].contiguous()
            solo, _ = _run(q[b:b + 1], k[b:b + 1], v[b:b + 1], H, D ** -0.5, wb, g, stat, impl="dense")
            assert torch.equal(solo[0], got[b]), f"image {b}"


# ------------------------------------------------------------------------------------------------------------------
# F. the std statistic at full UNet sizes and with mean(S) >> std(S)
# ------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("impl", IMPLS)
@pytest.mark.parametrize("N,H,D,T", [(4096, 8, 40, 77), (9216, 5, 64, 77), (4096, 8, 40, 231)])
def test_std_at_full_size(N, H, D, T, impl):
    q, k, v, w = _inputs(1, N, H, D, T, seed=N + D + T)
    ref, ref_st = _ref(q, k, v, H, D ** -0.5, [w[0].numpy()], G_STD, "std")
    got, st = _run(q, k, v, H, D ** -0.5, w, G_STD, "std", impl=impl)
    _check(got, st, ref, ref_st)


@pytest.mark.parametrize("impl", IMPLS)
@pytest.mark.parametrize("N,H,D,T", [(4096, 8, 40, 77), (1024, 8, 80, 231)])
def test_std_with_large_mean(N, H, D, T, impl):
    """Every q and k row shares a per-head component: S ~ 576 +- 17, so the variance is a small difference of large sums."""
    q, k, v, w = _inputs(1, N, H, D, T, seed=N + T + 5)
    gen = torch.Generator().manual_seed(N + T)
    u = torch.randn(H, D, generator=gen)
    u = (u / u.norm(dim=1, keepdim=True)).reshape(1, 1, H * D)
    q = (q.float() + 24.0 * u).half()
    k = (k.float() + 24.0 * u).half()
    qh = q[0].double().reshape(N, H, D).transpose(0, 1)
    kh = k[0].double().reshape(T, H, D).transpose(0, 1)
    s = qh @ kh.transpose(1, 2)
    assert (s.mean() / s.std()).item() >= 20.0
    ref, ref_st = _ref(q, k, v, H, D ** -0.5, [w[0].numpy()], G_STD, "std")
    got, st = _run(q, k, v, H, D ** -0.5, w, G_STD, "std", impl=impl)
    _check(got, st, ref, ref_st)


# ------------------------------------------------------------------------------------------------------------------
# G. key lengths below 77 at every head dim
# ------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("impl", IMPLS)
@pytest.mark.parametrize("stat", ["max", "std"])
@pytest.mark.parametrize("T", [1, 16, 41, 80])
@pytest.mark.parametrize("N,H,D", [(300, 5, 64), (256, 8, 80), (200, 4, 160)])
def test_short_key_lengths(N, H, D, T, stat, impl):
    q, k, v, w = _inputs(1, N, H, D, T, seed=T * 3 + D)
    g = G_MAX if stat == "max" else G_STD
    ref, ref_st = _ref(q, k, v, H, D ** -0.5, [w[0].numpy()], g, stat)
    got, st = _run(q, k, v, H, D ** -0.5, w, g, stat, impl=impl)
    _check(got, st, ref, ref_st)
