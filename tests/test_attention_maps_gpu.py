"""Attention recording on the GPU: the recording instances of the one-launch cross-attention kernel against an fp32
restatement of the per-region softmax mass, their bitwise properties, and the maps of whole runs against
oracle/attention_maps.py."""
import ctypes
import math

import pytest
import torch

import paint_with_words_sd_b200 as P
from oracle import loop as oracle_loop
from oracle.attention_maps import reference_attention_maps, token_regions
from paint_with_words_sd_b200 import _native, attention
from paint_with_words_sd_b200 import conditioning as C
from paint_with_words_sd_b200.pipeline import PwWSampler, region_adherence, region_coverage
from paint_with_words_sd_b200.scheduler import LMSDiscreteScheduler
from paint_with_words_sd_b200.synthetic import RandomTextEncoder, SimpleWordTokenizer
from paint_with_words_sd_b200.unet import UNetConfig, attention_modules, build_unet
from tests.fixtures import SETTINGS, color_map_image

pytestmark = pytest.mark.gpu

# Per-call mass tolerances (max abs, mass in [0, 1]).  The kernel multiplies P rounded to the element type and divides by
# the sum of exactly those rounded values; the fp32 restatement does neither, so the difference is the rounding of P:
# 2^-11 relative in fp16, 2^-8 in bf16, summed over up to 231 tokens of one region.
TOL = {torch.float16: 2e-3, torch.bfloat16: 1.6e-2}
# Loop level: the maps' rel RMSE bound of the other loop tests (fp16 UNet against the fp32 CPU loop), and adherence
LOOP_TOL, ADH_TOL = 3e-2, 1e-2

SD_SHAPES = [(4096, 8, 40), (1024, 8, 80), (256, 8, 160), (64, 8, 160),            # SD1.5 at 512
             (9216, 5, 64), (2304, 10, 64), (576, 20, 64), (144, 20, 64)]        # SD2.1 at 768
DEV = torch.device("cuda", 0)


def _inputs(B, N, H, D, T, dtype, seed):
    g = torch.Generator().manual_seed(seed)
    q = (torch.randn(B, N, H * D, generator=g) * 0.5).to(dtype)
    k = (torch.randn(B, T, H * D, generator=g) * 0.5).to(dtype)
    v = (torch.randn(B, T, H * D, generator=g) * 0.5).to(dtype)
    return q, k, v


def _maps(nbw, N, T, seed):
    g = torch.Generator().manual_seed(seed)
    w = torch.zeros(nbw, N, T)
    for i in range(nbw):
        w[i, :, 5 + i] = (torch.rand(N, generator=g) > 0.5).float() * 1.5
        w[i, :, 6 + i] = w[i, :, 5 + i]
        w[i, :, 11 + i] = (torch.rand(N, generator=g) > 0.7).float() * 0.6
    return w


def _ridx(Br, T, seed):
    """Random token -> slot rows (every slot 0..15 used, some tokens -1), in the cidx column layout."""
    g = torch.Generator().manual_seed(seed)
    owner = torch.randint(-1, 16, (Br, T), generator=g).to(torch.int8)
    k = C.key_chunks(T)
    row = torch.full((Br, 80 * k), -1, dtype=torch.int8)
    row[:, C._cidx_columns(T)] = owner
    return row, owner


def _call(q, k, v, H, w, idx_l, dtype, record=None, g=0.4 * math.log(8.0)):
    B = q.shape[0]
    kinds = torch.zeros(B, dtype=torch.int32, device=DEV)
    gs = torch.full((B,), g, dtype=torch.float32, device=DEV)
    idx = torch.tensor(idx_l, dtype=torch.int32, device=DEV)
    D = q.shape[2] // H
    has_map = w is not None and max(idx_l) >= 0
    return attention.cross_attention(q.to(DEV), k.to(DEV), v.to(DEV), H, D ** -0.5, w.to(DEV) if has_map else None,
                                     idx if has_map else None, kinds, gs, record=record)


def _oracle_mass(q, k, v, H, wb, owner, dtype, g=0.4 * math.log(8.0)):
    """fp32 [H, N, 16] mass of one image (wb [N, T] or None: unbiased), bias with the statistic rounded to `dtype`."""
    D = q.shape[-1] // H
    qh = q.float().reshape(-1, H, D).permute(1, 0, 2)
    kh = k.float().reshape(-1, H, D).permute(1, 0, 2)
    s = qh @ kh.transpose(1, 2)
    if wb is not None:
        stat = s.max().to(dtype).float()
        s = s + g * stat * wb
    p = (s * D ** -0.5).softmax(-1)
    mass = torch.zeros(H, q.shape[0], 16)
    for r in range(16):
        sel = owner.long() == r
        if sel.any():
            mass[..., r] = p[..., sel].sum(-1)
    return mass


def _record(B, Br, H, N, T, seed):
    ridx, owner = _ridx(Br, T, seed)
    acc = torch.zeros(Br, H, N, 16, dtype=torch.float32, device=DEV)
    return ridx.to(DEV), owner, acc


def _check_parity(B, N, H, D, T, dtype, idx_l, rec_l, seed=0):
    q, k, v = _inputs(B, N, H, D, T, dtype, seed)
    nbw = max(max(idx_l) + 1, 1)
    w = _maps(nbw, N, T, seed + 1)
    Br = max(rec_l) + 1
    ridx, owner, acc = _record(B, Br, H, N, T, seed + 2)
    rec_index = torch.tensor(rec_l, dtype=torch.int32, device=DEV)
    _call(q, k, v, H, w, idx_l, dtype, record=(ridx, rec_index, acc))
    torch.cuda.synchronize()
    acc = acc.cpu()
    err = 0.0
    for b in range(B):
        if rec_l[b] < 0:
            continue
        ref = _oracle_mass(q[b], k[b], v[b], H, w[idx_l[b]] if idx_l[b] >= 0 else None, owner[rec_l[b]], dtype)
        err = max(err, (acc[rec_l[b]] - ref).abs().max().item())
    assert err <= TOL[dtype], err
    for r in set(range(Br)) - {x for x in rec_l if x >= 0}:
        assert (acc[r] == 0).all()                         # records no image points to stay untouched


@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16])
@pytest.mark.parametrize("shape", SD_SHAPES, ids=lambda s: f"N{s[0]}_H{s[1]}_D{s[2]}")
def test_mass_matches_fp32_at_every_sd_level(shape, dtype):
    N, H, D = shape
    _check_parity(2, N, H, D, 77, dtype, [0, -1], [0, 1])          # cond (biased) + uncond, both recorded


@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16])
@pytest.mark.parametrize("T", [77, 154, 231])
@pytest.mark.parametrize("N", [1, 100, 333])
def test_mass_ragged_rows_and_long_contexts(N, T, dtype):
    _check_parity(4, N, 8, 40, T, dtype, [0, 1, -1, -1], [0, 1, 2, -1])


@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16])
@pytest.mark.parametrize("batch", ["biased", "unbiased", "mixed16"])
def test_mass_batches_and_splits(batch, dtype):
    L = _native.lib()
    L.pww_debug_set_fused_grid.argtypes = [ctypes.c_int]
    if batch == "biased":
        idx_l, rec_l = [0, 1, 2, 3], [3, 2, 1, 0]
    elif batch == "unbiased":
        idx_l, rec_l = [-1] * 4, [0, -1, 1, 2]
    else:
        idx_l, rec_l = [i if i < 8 else -1 for i in range(16)], list(range(16))
    try:
        # a small persistent grid: long job lists per CTA, and the C ABI halves the batch into several launches
        assert L.pww_debug_set_fused_grid(16) == 0
        _check_parity(len(idx_l), 1024, 8, 80, 77, dtype, idx_l, rec_l, seed=3)
    finally:
        L.pww_debug_set_fused_grid(0)


@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16])
@pytest.mark.parametrize("T", [77, 154, 231])
def test_all_tokens_in_one_slot_give_mass_one(T, dtype):
    B, N, H, D = 2, 333, 8, 64
    q, k, v = _inputs(B, N, H, D, T, dtype, 5)
    w = _maps(1, N, T, 6)
    ridx = torch.full((1, 80 * C.key_chunks(T)), -1, dtype=torch.int8)
    ridx[:, C._cidx_columns(T)] = 0
    acc = torch.zeros(1, H, N, 16, device=DEV)
    for idx_l in ([0, -1], [-1, 0]):                               # the recorded image biased, then unbiased
        acc.zero_()
        _call(q, k, v, H, w, idx_l, dtype, record=(ridx.to(DEV), torch.tensor([0, -1], dtype=torch.int32, device=DEV),
                                                   acc))
        a = acc.cpu()
        assert (a[..., 0] - 1).abs().max().item() <= 1e-5
        assert (a[..., 1:] == 0).all()


@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16])
def test_out_is_bitwise_the_plain_kernel_and_recording_is_deterministic(dtype):
    B, N, H, D, T = 6, 1024, 8, 80, 154
    q, k, v = _inputs(B, N, H, D, T, dtype, 7)
    w = _maps(3, N, T, 8)
    idx_l = [0, -1, 1, -1, 2, -1]
    ridx, _, acc1 = _record(B, B, H, N, T, 9)
    acc2 = torch.zeros_like(acc1)
    rec_index = torch.arange(B, dtype=torch.int32, device=DEV)
    plain = _call(q, k, v, H, w, idx_l, dtype)
    rec1 = _call(q, k, v, H, w, idx_l, dtype, record=(ridx, rec_index, acc1))
    rec2 = _call(q, k, v, H, w, idx_l, dtype, record=(ridx, rec_index, acc2))
    assert torch.equal(plain, rec1) and torch.equal(plain, rec2)
    assert torch.equal(acc1, acc2)
    # two calls into one buffer add up to the two single calls
    _call(q, k, v, H, w, idx_l, dtype, record=(ridx, rec_index, acc2))
    assert torch.equal(acc2, acc1 + acc1)


@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16])
def test_one_image_records_the_same_alone_or_in_a_batch_of_16(dtype):
    B, N, H, D, T = 16, 4096, 8, 40, 77
    q, k, v = _inputs(B, N, H, D, T, dtype, 11)
    w = _maps(8, N, T, 12)
    idx_l = [i if i < 8 else -1 for i in range(B)]
    ridx, _, acc = _record(B, B, H, N, T, 13)
    _call(q, k, v, H, w, idx_l, dtype, record=(ridx, torch.arange(B, dtype=torch.int32, device=DEV), acc))
    for b in (3, 12):                                               # a biased and an unbiased image
        one = torch.zeros(1, H, N, 16, device=DEV)
        _call(q[b:b + 1], k[b:b + 1], v[b:b + 1], H, w[idx_l[b]:idx_l[b] + 1] if idx_l[b] >= 0 else None,
              [0 if idx_l[b] >= 0 else -1], dtype, record=(ridx[b:b + 1].contiguous(),
                                                            torch.zeros(1, dtype=torch.int32, device=DEV), one))
        assert torch.equal(one[0], acc[b]), b


def test_recording_refuses_the_dense_path():
    B, N, H, D, T = 2, 64, 8, 40, 77
    q, k, v = _inputs(B, N, H, D, T, torch.float16, 14)
    ridx, _, acc = _record(B, B, H, N, T, 15)
    rec = (ridx, torch.arange(B, dtype=torch.int32, device=DEV), acc)
    old = attention.XATTN_IMPL
    try:
        attention.XATTN_IMPL = "dense"
        with pytest.raises(_native.NativeError, match="one-launch"):
            _call(q, k, v, H, _maps(1, N, T, 16), [0, -1], torch.float16, record=rec)
    finally:
        attention.XATTN_IMPL = old
    w = torch.zeros(1, N, T)
    for t in range(12):                                             # 12 distinct columns: no packed form
        w[0, :, t] = 0.1 * (t + 1) * (torch.arange(N) % (t + 2) == 0).float()
    with pytest.raises(_native.NativeError, match="dense"):
        _call(q, k, v, H, w, [0, -1], torch.float16, record=rec)


# ---- whole runs on the tiny UNet ----
SIZE, STEPS = 128, 4
WF = lambda w, sigma, qk: 0.4 * w * math.log(1 + sigma) * qk.max()      # noqa: E731
WF_ZERO = lambda w, sigma, qk: 0.0                                       # noqa: E731


def _scheduler():
    sch = LMSDiscreteScheduler(beta_start=0.00085, beta_end=0.012, beta_schedule="scaled_linear")
    sch.set_timesteps(STEPS)
    return sch


def _encode(cfg, device, chunks=1, repeat=1):
    s = SETTINGS["aurora"]
    _, sep, cond, uncond = C._encode_text_color_inputs(
        RandomTextEncoder(cfg.cross_attention_dim).to(device), SimpleWordTokenizer(), device,
        color_map_image("aurora", SIZE), dict(s["ctx"]), " ".join([s["prompt"]] * repeat), "", max_prompt_chunks=chunks)
    return sep, cond, uncond


def _latents(sch):
    return torch.randn(1, 4, SIZE // 8, SIZE // 8, generator=torch.manual_seed(0)) * sch.init_noise_sigma


def _extra():
    g = torch.Generator().manual_seed(9)
    mask = (torch.rand(1, 1, SIZE // 8, SIZE // 8, generator=g) > 0.5).float()
    return torch.cat([mask, torch.randn(1, 4, SIZE // 8, SIZE // 8, generator=g)], 1)


def _gpu_run(cfg, wf, record, use_graph, chunks, repeat, inpaint):
    unet = build_unet(cfg, seed=0, dtype=torch.float16, device="cuda")
    sch = _scheduler()
    _, cond, uncond = _encode(cfg, "cuda", chunks, repeat)
    P.patch_unet(unet)
    try:
        s = PwWSampler(unet, sch, [cond], [uncond], _latents(sch).cuda(), wf, 7.5, use_graph=use_graph,
                       extra_input=_extra().cuda() if inpaint else None, record_attention=record)
        out = s.run().float().cpu()
    finally:
        P.unpatch_all()
    return out, (s.attention_maps()[0] if record else None)


def _rel_rmse(a, b):
    return ((a - b).pow(2).mean().sqrt() / b.pow(2).mean().sqrt()).item()


LOOP_CASES = {"default": dict(), "zero": dict(wf=WF_ZERO), "two_chunks": dict(chunks=2, repeat=3),
              "inpaint": dict(inpaint=True)}


@pytest.mark.parametrize("case", sorted(LOOP_CASES))
def test_run_maps_match_the_oracle_and_latents_are_unchanged(case):
    kw = dict(dict(wf=WF, chunks=1, repeat=1, inpaint=False), **LOOP_CASES[case])
    cfg = UNetConfig.tiny(in_channels=9 if kw["inpaint"] else 4)
    for use_graph in (True, False):
        plain, _ = _gpu_run(cfg, kw["wf"], False, use_graph, kw["chunks"], kw["repeat"], kw["inpaint"])
        rec, maps = _gpu_run(cfg, kw["wf"], True, use_graph, kw["chunks"], kw["repeat"], kw["inpaint"])
        assert torch.equal(plain, rec), use_graph
    sep, cond, uncond = _encode(cfg, "cpu", kw["chunks"], kw["repeat"])
    unet = build_unet(cfg, seed=0)
    sch = _scheduler()
    ids = cond[C.REGION_INDEX_KEY]
    T = cond["CONTEXT_TENSOR"].shape[1]
    owner = ids[C._cidx_columns(T)].tolist()
    toks = C.chunk_prompt(SimpleWordTokenizer(), " ".join([SETTINGS["aurora"]["prompt"]] * kw["repeat"]),
                          [v.rpartition(",")[0] for v in SETTINGS["aurora"]["ctx"].values()], kw["chunks"])[0].tolist()
    assert owner == token_regions([lab for lab, _ in sep], toks)      # the row is the oracle's token rule
    _, ref = reference_attention_maps(unet, sch, cond, uncond, _latents(sch), kw["wf"], owner, len(sep),
                                      extra_input=_extra() if kw["inpaint"] else None)
    assert maps.shape == ref.shape == (5, SIZE // 8, SIZE // 8)
    assert _rel_rmse(maps, ref) <= LOOP_TOL
    cov = region_coverage(color_map_image("aurora", SIZE), SETTINGS["aurora"]["ctx"], (SIZE // 8, SIZE // 8))
    has = [bool((ids == r).any()) for r in range(5)]
    a, b = region_adherence(maps, cov, has), region_adherence(ref, cov, has)
    assert ((a - b).abs() <= ADH_TOL).all(), (a, b)


def test_restart_zeroes_the_maps_and_launches_are_unchanged():
    cfg = UNetConfig.tiny()
    unet = build_unet(cfg, seed=0, dtype=torch.float16, device="cuda")
    sch = _scheduler()
    _, cond, uncond = _encode(cfg, "cuda")
    P.patch_unet(unet)
    try:
        s = PwWSampler(unet, sch, [cond], [uncond], _latents(sch).cuda(), WF, 7.5, record_attention=True)
        plain = PwWSampler(unet, sch, [cond], [uncond], _latents(sch).cuda(), WF, 7.5)
        s.run(2)
        plain.run(2)
        first = s.attention_maps()[0]
        s.restart(_latents(sch).cuda())
        s.run(2)
        assert torch.equal(first, s.attention_maps()[0])
        assert s.native_launches_per_step == plain.native_launches_per_step
    finally:
        P.unpatch_all()


def test_public_api_returns_region_attention():
    a = SETTINGS["aurora"]
    tools = P.pww_load_tools("cuda:0", hf_model_path="synthetic:tiny")
    try:
        kw = dict(color_map_image=color_map_image("aurora", SIZE), input_prompt=a["prompt"], num_inference_steps=4,
                  device="cuda:0", preloaded_utils=tools, return_latents=True)
        plain = P.paint_with_words(color_context=dict(a["ctx"]), **kw)
        lat, att = P.paint_with_words(color_context=dict(a["ctx"]), return_attention_maps=True, **kw)
        _, att0 = P.paint_with_words(color_context=dict(a["ctx"]), return_attention_maps=True,
                                     weight_function=WF_ZERO, **kw)
        pairs = P.paint_with_words_batch([dict(color_context=a["ctx"], color_map_image=kw["color_map_image"],
                                               input_prompt=a["prompt"])] * 2, num_inference_steps=4, device="cuda:0",
                                         preloaded_utils=tools, return_latents=True, return_attention_maps=True)
    finally:
        P.unpatch_all()
    assert torch.equal(plain, lat)
    assert isinstance(att, P.RegionAttention)
    assert att.labels == [v.rpartition(",")[0] for v in a["ctx"].values()]
    assert att.maps.shape == att.coverage.shape == (5, SIZE // 8, SIZE // 8)
    assert ((att.adherence >= 0) & (att.adherence <= 1)).all()
    assert len(pairs) == 2 and all(isinstance(p_[1], P.RegionAttention) for p_ in pairs)
    # reported, not asserted: synthetic weights give no guarantee that the bias raises adherence
    print("adherence default:", [round(x, 4) for x in att.adherence.tolist()],
          "zero weight function:", [round(x, 4) for x in att0.adherence.tolist()])
