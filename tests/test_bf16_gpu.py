"""bf16 on the GPU: every native kernel family with bfloat16 activations against the oracles, the batching and view
invariances of the fp16 suite, the sampler kernels bitwise, the sampler loop and the public API with torch_dtype.

Tolerances are the fp16 suite's multiplied by 8, the ratio of the two formats' unit roundoffs (2^-9 / 2^-12), frozen
here:
  * statistic: relative 2^-7 (one bf16 ulp) against the bf16-emulating oracle;
  * cross-attention output vs the fp32 oracle: max|d| <= 1.6e-2 * max|out|; vs the bf16-emulating oracle: 1.2e-2;
  * self-attention: 1.6e-2 (2.4e-2 for the peaky-score case).
GroupNorm, GEGLU and add+LayerNorm are held per element to the bound of tests/unet_ops_bound.py against fp64.
The bf16-emulating oracle is `oracle.pww_oracle.attention_core` with bf16 rounding points in place of fp16 ones.  Each
check prints `BF16 <test> <measured> <bound>` (run pytest with -s to see the measured maxima).
"""
import math

import pytest
import torch

import paint_with_words_sd_b200 as P
from oracle import pww_oracle as O
from paint_with_words_sd_b200 import _native, fused_ops
from paint_with_words_sd_b200 import attention as A
from paint_with_words_sd_b200.pipeline import PwWSampler
from paint_with_words_sd_b200.unet import UNetConfig, build_unet
from tests import unet_ops_bound as U
from tests.fixtures import SETTINGS, color_map_image, moon_mask_image
from tests.test_per_image_settings_gpu import IMAGES, _encode, _latents, _scheduler, reference_loops  # noqa: F401
from tests.test_samplers_gpu import _bitwise_case
from tests.test_selfattn_gpu import SHAPES as SELF_SHAPES
from tests.test_xattn_gpu import IMPLS, RAGGED, SD15_256, SD15_512, SD21_768

pytestmark = pytest.mark.gpu
BF = torch.bfloat16


def _report(name, measured, bound):
    print(f"BF16 {name} {measured:.3e} {bound:.3e}")
    assert measured <= bound, (name, measured, bound)


# ---- oracles ---------------------------------------------------------------------------------------------------------
def _core(q, k, v, heads, scale, bias_fn, dtype):
    """oracle.pww_oracle.attention_core with the rounding points of an autocast to `dtype` (None = fp32)."""
    def r(t):
        return t.to(dtype).to(torch.float32) if dtype is not None else t
    q, k, v = r(q.float()), r(k.float()), r(v.float())
    qh, kh, vh = O._h2b(q, heads), O._h2b(k, heads), O._h2b(v, heads)
    s = r(torch.matmul(qh, kh.transpose(-1, -2)))
    bias = bias_fn(s.to(dtype) if dtype is not None else s) if bias_fn is not None else 0.0
    if isinstance(bias, torch.Tensor):
        s = (s + bias.float()) * scale
    else:
        s = r((s + bias) * scale)
    p = r(s.softmax(dim=-1))
    return O._b2h(r(torch.matmul(p, vh)), heads)


def _oracle(q, k, v, H, scale, w, g, stat, dtype):
    """Per image: output and the statistic (`max` / `std` of the scores as the dtype's autocast returns it)."""
    outs, stats = [], []
    for b in range(q.shape[0]):
        box = {}

        def bias_fn(s, b=b):
            m = s.max() if stat == "max" else s.std()
            box["m"] = float(m)
            return g * w[b] * m.float()
        outs.append(_core(q[b:b + 1], k[b:b + 1], v[b:b + 1], H, scale, bias_fn if w is not None else None, dtype))
        stats.append(box.get("m", 0.0))
    return torch.cat(outs, 0), stats


def _inputs(B, N, H, D, T, seed, spread=0.5):
    g = torch.Generator().manual_seed(seed)
    C = H * D
    q, k, v = [(torch.randn(B, L, C, generator=g) * spread).to(BF) for L in (N, T, T)]
    w = torch.zeros(B, N, T)
    for b in range(B):                      # sparse columns like the real maps, plus overlap
        for c in torch.randperm(T, generator=g)[:9]:
            w[b, :, c] += (torch.rand(N, generator=g) > 0.6).float() * float(torch.rand(1, generator=g) * 2)
    return q, k, v, w


def _xattn(q, k, v, H, scale, w=None, g=0.0, stat=_native.PWW_STAT_MAX, idx=None, impl="fused", gs=None):
    """cross_attention on the GPU; `stat` an int, or an int32 [B] kind tensor with `gs` the fp32 [B] G tensor."""
    old = A.XATTN_IMPL
    A.XATTN_IMPL = impl
    try:
        if gs is None:
            gs = torch.tensor([g], dtype=torch.float32)
        out, st = A.cross_attention(q.cuda(), k.cuda(), v.cuda(), H, scale, None if w is None else w.cuda(),
                                    None if idx is None else idx.cuda(),
                                    stat.cuda() if isinstance(stat, torch.Tensor) else stat, gs.cuda(),
                                    return_stats=True)
        torch.cuda.synchronize()
    finally:
        A.XATTN_IMPL = old
    assert out.dtype == BF
    return out.cpu(), (None if st is None else st.cpu())


def _gain(stat):
    return 0.4 * math.log(1 + 7.0) if stat == "max" else 0.5 * math.log(1 + 7.0 ** 2)


# ---- cross-attention -------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("impl", IMPLS)
@pytest.mark.parametrize("N,H,D", SD15_512 + SD15_256 + SD21_768 + RAGGED)
@pytest.mark.parametrize("T", [77, 154, 231])
@pytest.mark.parametrize("stat", ["max", "std"])
def test_bias_path_matches_oracles(N, H, D, T, stat, impl):
    if stat == "std" and N * H > 40000:
        pytest.skip("std covered at the smaller sizes; max covers the large ones (as in the fp16 suite)")
    q, k, v, w = _inputs(1, N, H, D, T, seed=N * 131 + D + T)
    scale, g = D ** -0.5, _gain(stat)
    got, st = _xattn(q, k, v, H, scale, w, g, _native.PWW_STAT_MAX if stat == "max" else _native.PWW_STAT_STD,
                     impl=impl)
    ref_bf, st_bf = _oracle(q, k, v, H, scale, w, g, stat, BF)
    ref32, _ = _oracle(q, k, v, H, scale, w, g, stat, None)
    tag = f"xattn-{impl}-{N}x{H}x{D}-T{T}-{stat}"
    if N * H * T > 1:
        _report(tag + "-stat", abs(float(st[0]) - st_bf[0]) / abs(st_bf[0]), 2 ** -7)
    amax = ref32.abs().max().item()
    _report(tag + "-vs-bf16", (got.float() - ref_bf).abs().max().item() / amax, 1.2e-2)
    _report(tag + "-vs-fp32", (got.float() - ref32).abs().max().item() / amax, 1.6e-2)


@pytest.mark.parametrize("impl", IMPLS)
@pytest.mark.parametrize("stat", ["max", "std"])
def test_large_scores_stay_finite(stat, impl):
    """Scores above 2e5, where an fp16 statistic is inf and the bias of a map's zero entries 0 * inf = NaN: finite, and
    within the fp32 oracle's tolerance.  The map weighs every token of the painted rows equally, so the output does not
    depend on the last bits of the huge bias, and is zero on the other rows."""
    N, H, D, T = 1024, 8, 40, 77
    g = torch.Generator().manual_seed(5)
    q, k, v = [(torch.randn(1, L, H * D, generator=g) * s).to(BF) for L, s in ((N, 100.0), (T, 100.0), (T, 0.5))]
    w = torch.zeros(1, N, T)
    w[0, : N // 2] = 1.0
    s_max = torch.matmul(O._h2b(q.float(), H), O._h2b(k.float(), H).transpose(-1, -2)).max().item()
    assert s_max > 2e5, s_max
    scale, gain = D ** -0.5, _gain(stat)
    ref32, st32 = _oracle(q, k, v, H, scale, w, gain, stat, None)
    got, st = _xattn(q, k, v, H, scale, w, gain, _native.PWW_STAT_MAX if stat == "max" else _native.PWW_STAT_STD,
                     impl=impl)
    assert torch.isfinite(got.float()).all() and math.isfinite(float(st[0]))
    _report(f"large-scores-{impl}-{stat}-stat", abs(float(st[0]) - st32[0]) / abs(st32[0]), 2 ** -7)
    _report(f"large-scores-{impl}-{stat}", (got.float() - ref32).abs().max().item() / ref32.abs().max().item(), 1.6e-2)


@pytest.mark.parametrize("impl", IMPLS)
@pytest.mark.parametrize("B", [2, 40])
def test_mixed_multi_batch_equals_solo_launches(B, impl):
    """Mixed kinds and G in one `_multi_bf16` launch (B = 40 splits it): every image bitwise equals its solo launch."""
    N, H, D, T = 256, 8, 40, 77
    q, k, v, w = _inputs(B, N, H, D, T, seed=B)
    g = torch.Generator().manual_seed(B + 1)
    kinds = torch.randint(0, 2, (B,), generator=g, dtype=torch.int32)
    gs = torch.rand(B, generator=g) * 2 + 0.1
    idx = torch.arange(B, dtype=torch.int32)
    idx[1::3] = -1                                  # some images unbiased
    got, st = _xattn(q, k, v, H, D ** -0.5, w, stat=kinds, idx=idx, impl=impl, gs=gs)
    for b in range(B):
        biased = int(idx[b]) >= 0
        solo, sst = _xattn(q[b:b + 1], k[b:b + 1], v[b:b + 1], H, D ** -0.5, w[b:b + 1] if biased else None,
                           float(gs[b]), int(kinds[b]), impl=impl)
        assert torch.equal(solo[0], got[b]), b
        assert float(st[b]) == (float(sst[0]) if biased else 0.0), b


@pytest.mark.parametrize("impl", IMPLS)
def test_uniform_batches_views_and_broadcast_contexts_are_bitwise_invariant(impl):
    N, H, D, T, B = 1024, 8, 80, 77, 3
    C, scale = H * D, D ** -0.5
    q, k, v, w = _inputs(B, N, H, D, T, seed=11)
    # all-biased and all-unbiased batches against solo launches
    allb, _ = _xattn(q, k, v, H, scale, w, 0.9, idx=torch.arange(B, dtype=torch.int32), impl=impl)
    allu, _ = _xattn(q, k, v, H, scale, impl=impl)
    for b in range(B):
        assert torch.equal(allb[b], _xattn(q[b:b + 1], k[b:b + 1], v[b:b + 1], H, scale, w[b:b + 1], 0.9,
                                           impl=impl)[0][0]), b
        assert torch.equal(allu[b], _xattn(q[b:b + 1], k[b:b + 1], v[b:b + 1], H, scale, impl=impl)[0][0]), b
    # strided views: q a column slice of a wider buffer, k / v slices of one [B, T, 2C] buffer
    qbuf = torch.cat([q, torch.zeros_like(q)], -1)
    kv = torch.cat([k, v], -1)
    strided, _ = _xattn(qbuf[..., :C], kv[..., :C], kv[..., C:], H, scale, w, 0.9,
                        idx=torch.arange(B, dtype=torch.int32), impl=impl)
    assert torch.equal(strided, allb)
    # stride-0 (broadcast) contexts against contiguous copies
    kb, vb = k[:1].expand(B, -1, -1), v[:1].expand(B, -1, -1)
    bcast, _ = _xattn(q, kb, vb, H, scale, w, 0.9, idx=torch.arange(B, dtype=torch.int32), impl=impl)
    copy, _ = _xattn(q, kb.contiguous(), vb.contiguous(), H, scale, w, 0.9, idx=torch.arange(B, dtype=torch.int32),
                     impl=impl)
    assert torch.equal(bcast, copy)


# ---- self-attention --------------------------------------------------------------------------------------------------
def _native_self_attention(q, k, v, H, scale):
    old = A.SELF_ATTN_IMPL
    A.SELF_ATTN_IMPL = "native"
    try:
        before = _native.launch_count
        out = A.self_attention(q.cuda(), k.cuda(), v.cuda(), H, scale)
        assert _native.launch_count == before + 1 and out.dtype == BF
    finally:
        A.SELF_ATTN_IMPL = old
    torch.cuda.synchronize()
    return out.float().cpu()


@pytest.mark.parametrize("N,H,D", SELF_SHAPES + [(9216, 5, 64)])
def test_self_attention_matches_oracle(N, H, D):
    g = torch.Generator().manual_seed(N + D)
    q, k, v = [(torch.randn(2 if N <= 1024 else 1, N, H * D, generator=g) * 0.5).to(BF) for _ in range(3)]
    got = _native_self_attention(q, k, v, H, D ** -0.5)
    ref = torch.cat([O.attention_core(q[b:b + 1].float(), k[b:b + 1].float(), v[b:b + 1].float(), H, D ** -0.5)
                     for b in range(q.shape[0])], 0)
    _report(f"self-{N}x{H}x{D}", (got - ref).abs().max().item() / ref.abs().max().item(), 1.6e-2)


def test_self_attention_peaky_scores():
    N, H, D = 512, 2, 64
    g = torch.Generator().manual_seed(1)
    q, k, v = [(torch.randn(1, N, H * D, generator=g) * 0.5) for _ in range(3)]
    k = k * torch.linspace(0.2, 6.0, N)[None, :, None]
    q, k, v = q.to(BF), k.to(BF), v.to(BF)
    got = _native_self_attention(q, k, v, H, D ** -0.5)
    ref = O.attention_core(q.float(), k.float(), v.float(), H, D ** -0.5)
    _report("self-peaky", (got - ref).abs().max().item() / ref.abs().max().item(), 2.4e-2)


# ---- UNet ops --------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("C,HW,G", [(320, 64, 32), (640, 32, 32), (1280, 16, 32), (1280, 8, 32), (2560, 8, 32),
                                    (1920, 16, 32), (960, 32, 32), (160, 16, 8), (480, 7, 8)])
@pytest.mark.parametrize("silu,with_add", [(True, False), (True, True), (False, False)])
def test_group_norm_nhwc(C, HW, G, silu, with_add):
    g = torch.Generator().manual_seed(C + HW)
    B = 2
    x = (torch.randn(B, C, HW, HW, generator=g) * 1.5 + 0.3).to(BF)
    gn = torch.nn.GroupNorm(G, C, eps=1e-5)
    gn.weight.data = torch.randn(C, generator=g) * 0.5 + 1.0
    gn.bias.data = torch.randn(C, generator=g) * 0.2
    add = (torch.randn(B, C, generator=g) * 0.5).to(BF) if with_add else None
    gn_b = gn.to(BF).cuda()
    got = fused_ops.group_norm_nhwc(x.cuda().contiguous(memory_format=torch.channels_last), gn_b,
                                    None if add is None else add.cuda(), silu=silu)
    assert got.dtype == BF and got.is_contiguous(memory_format=torch.channels_last)
    ref, terms = U.gn_reference(x.cuda().flatten(2).transpose(1, 2), gn_b.weight, gn_b.bias, G, 1e-5,
                                None if add is None else add.cuda(), silu)
    worst = U.check_within(got.flatten(2).transpose(1, 2), ref, terms, BF, U.K_GN, f"gn {C} {HW} {G}")
    print(f"BF16 groupnorm-{C}-{HW}-{G}-{silu}-{with_add} worst {worst:.3f} of the allowance")


@pytest.mark.parametrize("M,I", [(2 * 4096, 1280), (2 * 64, 5120), (3, 8), (77, 2560)])
def test_geglu(M, I):
    g = torch.Generator().manual_seed(M + I)
    h = (torch.randn(M, 2 * I, generator=g) * 2.0).to(BF)
    ref, terms = U.geglu_reference(h)
    got = fused_ops.geglu(h.cuda())
    assert got.dtype == BF
    worst = U.check_within(got.cpu(), ref, terms, BF, U.K_GEGLU, f"geglu {M} {I}")
    print(f"BF16 geglu-{M}-{I} worst {worst:.3f} of the allowance")


@pytest.mark.parametrize("M,C", [(2 * 4096, 320), (2 * 1024, 640), (2 * 256, 1280), (5, 1280), (3, 8), (7, 2048)])
@pytest.mark.parametrize("with_res", [True, False])
def test_add_layer_norm(M, C, with_res):
    g = torch.Generator().manual_seed(M + C)
    x = (torch.randn(M, C, generator=g) * 2.0).to(BF).cuda()
    res = (torch.randn(M, C, generator=g) * 2.0).to(BF).cuda() if with_res else None
    ln = torch.nn.LayerNorm(C)
    ln.weight.data = torch.randn(C, generator=g) * 0.5 + 1.0
    ln.bias.data = torch.randn(C, generator=g) * 0.2
    ln_b = ln.to(BF).cuda()
    s_ref = x + res if with_res else x                     # a bf16 torch add
    y_ref, terms = U.ln_reference(s_ref, ln_b.weight, ln_b.bias, ln.eps)
    s, y = fused_ops.add_layer_norm(x, res, ln_b)
    assert torch.equal(s, s_ref) and y.dtype == BF          # the residual stream is bit-identical
    worst = U.check_within(y, y_ref, terms, BF, U.K_LN, f"add-layernorm {M} {C}")
    print(f"BF16 add-layernorm-{M}-{C}-{with_res} worst {worst:.3f} of the allowance")


# ---- sampler kernels -------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("sampler", ["lms", "euler", "euler_a", "dpmpp_2m"])
@pytest.mark.parametrize("hw", [(64, 64), (15, 17)], ids=["64x64", "15x17"])
@pytest.mark.parametrize("inpaint", [False, True], ids=["txt2img", "inpaint"])
def test_native_step_is_bitwise_equal_to_torch(sampler, hw, inpaint):
    """UNet input == (x * scale).to(bfloat16) in rows i and m + i, and the update == the step form as torch ops with
    a bf16 eps, every step (channels-last eps; 15x17 takes the one-pixel path)."""
    _bitwise_case(sampler, 2, hw, inpaint, "channels_last", BF, steps=12)


# ---- loop and API ----------------------------------------------------------------------------------------------------
def _sampler(unet, cfg, images, use_graph, seeds=None):
    """One PwWSampler over `images` (entries of IMAGES); image j's latents come from seed seeds[j] (default: j)."""
    sch = _scheduler()
    enc = [_encode(cfg, name, "cuda") for name, _, _ in images]
    lat = torch.cat([_latents(i, sch) for i in (seeds or range(len(images)))], 0).cuda()
    return PwWSampler(unet, sch, [c for c, _ in enc], [u for _, u in enc], lat, [f for _, f, _ in images],
                      [g for _, _, g in images], use_graph=use_graph)


def _rel_rmse(a, b):
    return ((a - b).pow(2).mean().sqrt() / b.pow(2).mean().sqrt()).item()


def test_bf16_sampler_matches_reference_loop_beside_fp16(reference_loops):
    cfg = UNetConfig.tiny()
    runs, launches = {}, {}
    try:
        for dt in (torch.float16, BF):
            unet = build_unet(cfg, seed=0, dtype=dt, device="cuda")
            P.patch_unet(unet)
            s = _sampler(unet, cfg, IMAGES, use_graph=True)
            runs[dt] = s.run().float().cpu()
            launches[dt] = s.native_launches_per_step
            if dt == BF:
                eager = _sampler(unet, cfg, IMAGES, use_graph=False).run().float().cpu()
                assert torch.equal(eager, runs[BF])           # graph on and off give the same bits
                solo = [_sampler(unet, cfg, [img], use_graph=False, seeds=[i]).run().float().cpu()
                        for i, img in enumerate(IMAGES[:2])]
                pair = _sampler(unet, cfg, IMAGES[:2], use_graph=False).run().float().cpu()
                for i in range(2):
                    d = (pair[i] - solo[i][0]).abs().max().item()
                    _report(f"sampler-pair-vs-solo-{i}", d / solo[i].abs().max().item(), 2e-2)
    finally:
        P.unpatch_all()
    assert launches[BF] == launches[torch.float16] and launches[BF] > 2     # no route falls back to torch
    for i, ref in enumerate(reference_loops):
        print(f"BF16 loop-rel-rmse image {i}: fp16 {_rel_rmse(runs[torch.float16][i], ref[0]):.3e} "
              f"bf16 {_rel_rmse(runs[BF][i], ref[0]):.3e}")
        assert torch.isfinite(runs[BF][i]).all()
        _report(f"loop-rel-rmse-{i}", _rel_rmse(runs[BF][i], ref[0]), 0.1)


def test_public_api_with_torch_dtype_bf16():
    size = 128
    a, c = SETTINGS["aurora"], SETTINGS["cat_dog"]
    try:
        lat = P.paint_with_words(color_context=a["ctx"], color_map_image=color_map_image("aurora", size),
                                 input_prompt=a["prompt"], num_inference_steps=3, device="cuda:0",
                                 hf_model_path="synthetic:tiny", torch_dtype=BF, return_latents=True)
        assert lat.shape == (1, 4, size // 8, size // 8) and torch.isfinite(lat).all()
        img = P.paint_with_words(color_context=a["ctx"], color_map_image=color_map_image("aurora", size),
                                 input_prompt=a["prompt"], num_inference_steps=2, device="cuda:0",
                                 hf_model_path="synthetic:tiny", torch_dtype=BF)
        assert img.size == (size, size)
        lat = P.paint_with_words_inpaint(color_context=a["ctx"], color_map_image=color_map_image("aurora", size),
                                         mask_image=moon_mask_image(size), init_image=color_map_image("aurora", size),
                                         input_prompt=a["prompt"], num_inference_steps=3, device="cuda:0",
                                         hf_model_path="synthetic:tiny-inpaint", torch_dtype=BF, return_latents=True)
        assert lat.shape == (1, 4, size // 8, size // 8) and torch.isfinite(lat).all()
        entries = [dict(color_context=a["ctx"], color_map_image=color_map_image("aurora", size), input_prompt=a["prompt"]),
                   dict(color_context=c["ctx"], color_map_image=color_map_image("cat_dog", size), input_prompt=c["prompt"],
                        seed=1)]
        lats = P.paint_with_words_batch(entries, num_inference_steps=3, device="cuda:0", hf_model_path="synthetic:tiny",
                                        torch_dtype=BF, return_latents=True)
        assert len(lats) == 2 and all(x.shape == (1, 4, size // 8, size // 8) and torch.isfinite(x).all() for x in lats)
        imgs = P.paint_with_words_batch(entries, num_inference_steps=2, device="cuda:0", hf_model_path="synthetic:tiny",
                                        torch_dtype=BF)
        assert [im.size for im in imgs] == [(size, size)] * 2
    finally:
        P.unpatch_all()
