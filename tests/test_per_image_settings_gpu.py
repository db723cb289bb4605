"""Per-image weight functions and guidance scales on the GPU.

Kernels: a batch whose images take different statistic kinds and G(sigma) in ONE `_multi` launch gives every image
exactly (bitwise) what a solo launch of the existing entry point with that image's settings gives, on the one-launch
kernel and on the dense pair, at every SD shape and key length; the uniform `_multi` launch equals the existing entry
bitwise; the mixed batch matches the fp32 oracle with the tolerances of test_xattn_gpu.py.  Loop: a sampler whose
images have their own weight functions and guidance scales matches the reference loop run per image, and solo
samplers; the batch API matches `paint_with_words` per entry."""
import math

import pytest
import torch

import paint_with_words_sd_b200 as P
from oracle import loop as oracle_loop
from paint_with_words_sd_b200 import _native
from paint_with_words_sd_b200 import attention as A
from paint_with_words_sd_b200 import conditioning as C
from paint_with_words_sd_b200.pipeline import PwWSampler
from paint_with_words_sd_b200.scheduler import LMSDiscreteScheduler
from paint_with_words_sd_b200.synthetic import RandomTextEncoder, SimpleWordTokenizer
from paint_with_words_sd_b200.unet import UNetConfig, attention_modules, build_unet
from tests.fixtures import SETTINGS, color_map_image
from tests.test_xattn_gpu import IMPLS, SD15_256, SD15_512, SD21_768, _inputs, _oracle

pytestmark = pytest.mark.gpu
MAX, STD = _native.PWW_STAT_MAX, _native.PWW_STAT_STD
KEYS = [77, 154, 231]


def _xa(q, k, v, H, scale, w, idx, stat, g, impl):
    """One cross_attention call.  stat/g: an int kind and a float (existing entry points) or per-image lists (the
    `_multi` entry points).  Returns the fp16 output and the statistics on the host."""
    dev = "cuda"
    if isinstance(stat, list):
        stat = torch.tensor(stat, dtype=torch.int32, device=dev)
        gs = torch.tensor(g, dtype=torch.float32, device=dev)
    else:
        gs = torch.tensor([g], dtype=torch.float32, device=dev)
    old = A.XATTN_IMPL
    A.XATTN_IMPL = impl
    try:
        out, st = A.cross_attention(q.to(dev), k.to(dev), v.to(dev), H, scale, None if w is None else w.to(dev),
                                    None if idx is None else torch.tensor(idx, dtype=torch.int32, device=dev), stat, gs,
                                    return_stats=True)
        torch.cuda.synchronize()
    finally:
        A.XATTN_IMPL = old
    return out.cpu(), (None if st is None else st.cpu())


def _assert_each_image_equals_its_solo_launch(q, k, v, H, scale, w, idx, kinds, g, impl):
    got, st = _xa(q, k, v, H, scale, w, idx, kinds, g, impl)
    for b in range(q.shape[0]):
        one = slice(b, b + 1)
        if idx[b] >= 0:
            kind = STD if kinds[b] == STD else MAX
            solo, st_solo = _xa(q[one], k[one], v[one], H, scale, w[idx[b]:idx[b] + 1], None, kind, g[b], impl)
            assert float(st[b]) == float(st_solo[0]), (b, float(st[b]), float(st_solo[0]))
        else:
            solo, _ = _xa(q[one], k[one], v[one], H, scale, None, None, MAX, 0.0, impl)
            assert float(st[b]) == 0.0
        assert torch.equal(got[b], solo[0]), b


@pytest.mark.parametrize("impl", IMPLS)
@pytest.mark.parametrize("N,H,D", SD15_512 + SD15_256 + SD21_768)
@pytest.mark.parametrize("T", KEYS)
def test_mixed_launch_equals_solo_launches(T, N, H, D, impl):
    """Three cond images (max, std, and kind 7, which means max) with distinct G values on maps in reverse order, plus
    three uncond images whose kind and G entries (std, 100) must be ignored."""
    m = 3
    q, k, v, w = _inputs(2 * m, N, H, D, T, seed=N + 7 * D + T)
    q[1] *= 2.0                                      # different statistics per image
    idx = [m - 1 - b for b in range(m)] + [-1] * m
    kinds = [MAX, STD, 7] + [STD] * m
    g = [0.3 + 0.45 * b for b in range(m)] + [100.0] * m
    _assert_each_image_equals_its_solo_launch(q, k, v, H, D ** -0.5, w[:m].contiguous(), idx, kinds, g, impl)


@pytest.mark.parametrize("impl", IMPLS)
@pytest.mark.parametrize("N,H,D", [(256, 8, 40), (64, 8, 160)])
@pytest.mark.parametrize("T", [77, 154])
def test_large_mixed_batch_equals_solo_launches(T, N, H, D, impl):
    """B = 40: the one-launch kernel splits the batch at 32 images, so the kind and G arrays are read at an offset.
    Map indices are a permutation of 0..39 (many above 31); every fifth image is unbiased."""
    B = 40
    q, k, v, w = _inputs(B, N, H, D, T, seed=B + N + T)
    idx = [-1 if b % 5 == 4 else (7 * b) % B for b in range(B)]
    kinds = [STD if b % 3 == 0 else MAX for b in range(B)]
    g = [0.2 + 0.05 * b for b in range(B)]
    _assert_each_image_equals_its_solo_launch(q, k, v, H, D ** -0.5, w, idx, kinds, g, impl)


@pytest.mark.parametrize("impl", IMPLS)
@pytest.mark.parametrize("stat", [MAX, STD])
@pytest.mark.parametrize("N,H,D", [(4096, 8, 40), (1024, 8, 80), (576, 20, 64), (64, 8, 160)])
@pytest.mark.parametrize("T", KEYS)
def test_uniform_multi_launch_equals_the_existing_entry(T, N, H, D, stat, impl):
    q, k, v, w = _inputs(3, N, H, D, T, seed=3 * N + D + T)
    idx = [1, -1, 0]
    g = 0.4 * math.log(1 + 5.0)
    ref, st_ref = _xa(q, k, v, H, D ** -0.5, w[:2].contiguous(), idx, stat, g, impl)
    got, st = _xa(q, k, v, H, D ** -0.5, w[:2].contiguous(), idx, [stat] * 3, [g] * 3, impl)
    assert torch.equal(got, ref) and torch.equal(st, st_ref)


def _stat64(q, k, H, kind):
    """The statistic in float64 over the fp16-rounded scores of one image, rounded to fp16 (unbiased std)."""
    N, T, D = q.shape[1], k.shape[1], q.shape[2] // H
    s = torch.einsum("nhd,thd->hnt", q[0].double().view(N, H, D), k[0].double().view(T, H, D)).half().double()
    r = s.max() if kind == MAX else s.std()
    return float(r.half())


@pytest.mark.parametrize("impl", IMPLS)
@pytest.mark.parametrize("N,H,D", [(4096, 8, 40), (1024, 8, 80), (576, 20, 64), (64, 8, 160)])
@pytest.mark.parametrize("T", [77, 231])
def test_mixed_launch_matches_oracle(T, N, H, D, impl):
    """[cond max, cond std, uncond] against the fp32 oracle per image: statistic rel 2^-10 (float64 over fp16 scores),
    output max|d| <= 2e-3 * max|out|."""
    q, k, v, w = _inputs(3, N, H, D, T, seed=5 * N + D + T)
    scale = D ** -0.5
    idx = [0, 1, -1]
    kinds = [MAX, STD, MAX]
    g = [0.4 * math.log(1 + 7.0), 0.5 * math.log(1 + 7.0 ** 2), 0.0]
    got, st = _xa(q, k, v, H, scale, w[:2].contiguous(), idx, kinds, g, impl)
    got = got.float()
    for b in range(3):
        one = slice(b, b + 1)
        if idx[b] < 0:
            ref32, _ = _oracle(q[one], k[one], v[one], H, scale, None, 0.0, "max", emulate=False)
            assert float(st[b]) == 0.0
        else:
            name = "max" if kinds[b] == MAX else "std"
            wb = w[idx[b]:idx[b] + 1]
            ref32, _ = _oracle(q[one], k[one], v[one], H, scale, wb, g[b], name, emulate=False)
            st64 = _stat64(q[one], k[one], H, kinds[b])
            assert abs(float(st[b]) - st64) <= 2 ** -10 * abs(st64) + 1e-6, (b, float(st[b]), st64)
        assert (got[b] - ref32[0]).abs().max().item() <= 2e-3 * ref32.abs().max().item(), b


# ---------------------------------------------------------------------------------------------------------------------
# the loop
# ---------------------------------------------------------------------------------------------------------------------
WF_MAX = lambda w, sigma, qk: 0.4 * w * math.log(1 + sigma) * qk.max()          # noqa: E731
WF_STD2 = lambda w, sigma, qk: 0.4 * w * math.log(1 + sigma ** 2) * qk.std()    # noqa: E731
WF_ZERO = lambda w, sigma, qk: 0.0                                               # noqa: E731
# (colour map, weight function, guidance scale); image i starts from seed i
IMAGES = [("aurora", WF_MAX, 7.5), ("cat_dog", WF_STD2, 5.0), ("aurora", WF_ZERO, 9.0)]
SIZE, STEPS = 128, 4


def _scheduler():
    sch = LMSDiscreteScheduler(beta_start=0.00085, beta_end=0.012, beta_schedule="scaled_linear")
    sch.set_timesteps(STEPS)
    return sch


def _encode(cfg, name, device):
    tok, enc = SimpleWordTokenizer(), RandomTextEncoder(cfg.cross_attention_dim).to(device)
    s = SETTINGS[name]
    _, _, cond, uncond = C._encode_text_color_inputs(enc, tok, device, color_map_image(name, SIZE), dict(s["ctx"]),
                                                     s["prompt"], "")
    return cond, uncond


def _latents(i, sch):
    return torch.randn(1, 4, SIZE // 8, SIZE // 8, generator=torch.manual_seed(i)) * sch.init_noise_sigma


@pytest.fixture(scope="module")
def reference_loops():
    """The reference loop (two batch-1 fp32 CPU forwards per step, oracle attention) for every image, each with its own
    weight function and guidance scale."""
    cfg = UNetConfig.tiny()
    unet = build_unet(cfg, seed=0)
    refs = []
    try:
        oracle_loop.patch_with_oracle(unet)
        for i, (name, wf, cfg_scale) in enumerate(IMAGES):
            cond, uncond = _encode(cfg, name, "cpu")
            sch = _scheduler()
            refs.append(oracle_loop.reference_denoise_loop(unet, sch, cond, uncond, _latents(i, sch), wf, cfg_scale))
    finally:
        cls = attention_modules(unet)[0].__class__
        if "__call__" in cls.__dict__:
            delattr(cls, "__call__")
    return refs


def _gpu_sampler(unet, cfg, images, use_graph, weight_function=None, guidance_scale=None):
    sch = _scheduler()
    enc = [_encode(cfg, name, "cuda") for name, _, _ in images]
    lat = torch.cat([_latents(i, sch) for i in range(len(images))], 0).cuda()
    wf = [f for _, f, _ in images] if weight_function is None else weight_function
    gs = [g for _, _, g in images] if guidance_scale is None else guidance_scale
    return PwWSampler(unet, sch, [c for c, _ in enc], [u for _, u in enc], lat, wf, gs, use_graph=use_graph)


@pytest.mark.parametrize("use_graph", [False, True])
def test_sampler_with_per_image_settings_matches_reference_and_solo_runs(use_graph, reference_loops):
    cfg = UNetConfig.tiny()
    unet = build_unet(cfg, seed=0, dtype=torch.float16, device="cuda")
    try:
        P.patch_unet(unet)
        out = _gpu_sampler(unet, cfg, IMAGES, use_graph).run().float().cpu()
        solo = []
        for i, (name, wf, cfg_scale) in enumerate(IMAGES):
            sch = _scheduler()
            cond, uncond = _encode(cfg, name, "cuda")
            solo.append(PwWSampler(unet, sch, [cond], [uncond], _latents(i, sch).cuda(), wf, cfg_scale,
                                   use_graph=False).run().float().cpu())
    finally:
        P.unpatch_all()
    for i, ref in enumerate(reference_loops):
        rel_rmse = ((out[i] - ref[0]).pow(2).mean().sqrt() / ref.pow(2).mean().sqrt()).item()
        assert torch.isfinite(out[i]).all() and rel_rmse < 3e-2, (i, rel_rmse)
        d = (out[i] - solo[i][0]).abs().max().item()
        assert d <= 2e-2 * solo[i].abs().max().item(), (i, d)
    # the settings matter: image 0 and image 2 share map, prompt and UNet and differ only in seed and settings
    assert not torch.allclose(out[0], out[2])


def test_per_image_settings_keep_one_launch_per_attention_call():
    cfg = UNetConfig.tiny()
    unet = build_unet(cfg, seed=0, dtype=torch.float16, device="cuda")
    try:
        P.patch_unet(unet)
        mixed = _gpu_sampler(unet, cfg, IMAGES, use_graph=True)
        mixed.run(1)
        uniform = _gpu_sampler(unet, cfg, IMAGES, use_graph=True, weight_function=WF_MAX, guidance_scale=7.5)
        uniform.run(1)
    finally:
        P.unpatch_all()
    assert mixed.native_launches_per_step is not None and mixed.native_launches_per_step > 0
    assert mixed.native_launches_per_step == uniform.native_launches_per_step


def test_batch_api_matches_paint_with_words_per_entry():
    a, c = SETTINGS["aurora"], SETTINGS["cat_dog"]
    entries = [
        dict(color_context=a["ctx"], color_map_image=color_map_image("aurora", 128), input_prompt=a["prompt"], seed=0,
             weight_function=WF_MAX),
        dict(color_context=c["ctx"], color_map_image=color_map_image("cat_dog", 192), input_prompt=c["prompt"], seed=1,
             weight_function=WF_STD2, guidance_scale=5.0),
        dict(color_context=a["ctx"], color_map_image=color_map_image("aurora", 128), input_prompt=a["prompt"], seed=2,
             weight_function=WF_ZERO, guidance_scale=9.0),
    ]
    tools = P.pww_load_tools("cuda:0", hf_model_path="synthetic:tiny")
    try:
        got = P.paint_with_words_batch(entries, num_inference_steps=3, device="cuda:0", preloaded_utils=tools,
                                       return_latents=True)
        refs = [P.paint_with_words(**dict(e, color_context=dict(e["color_context"])), num_inference_steps=3,
                                   device="cuda:0", preloaded_utils=tools, return_latents=True) for e in entries]
        images = P.paint_with_words_batch(entries, num_inference_steps=2, device="cuda:0", preloaded_utils=tools)
    finally:
        P.unpatch_all()
    assert [tuple(x.shape) for x in got] == [(1, 4, 16, 16), (1, 4, 24, 24), (1, 4, 16, 16)]
    for i, (x, ref) in enumerate(zip(got, refs)):
        d = (x.float() - ref.float()).abs().max().item()
        assert torch.isfinite(x).all() and d <= 2e-2 * ref.abs().max().item(), (i, d)
    assert [im.size for im in images] == [(128, 128), (192, 192), (128, 128)]
