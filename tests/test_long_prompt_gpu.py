"""Long prompts on the GPU: cross-attention over 2 / 3 CLIP chunks (T = 154, 231) through the C ABI against the oracle,
with the tolerances of test_xattn_gpu.py (statistic rel 2^-10; 2e-3 * max|out| vs fp32; 1.5e-3 * max|out| vs the
fp16-emulating oracle), and the denoising loop with a 2-chunk prompt against the reference loop."""
import math

import pytest
import torch

import paint_with_words_sd_b200 as P
from oracle import loop as oracle_loop
from oracle import pww_oracle as O
from paint_with_words_sd_b200 import _native
from paint_with_words_sd_b200 import attention as A
from paint_with_words_sd_b200 import conditioning as C
from paint_with_words_sd_b200.pipeline import PwWSampler
from paint_with_words_sd_b200.scheduler import LMSDiscreteScheduler
from paint_with_words_sd_b200.synthetic import RandomTextEncoder, SimpleWordTokenizer
from paint_with_words_sd_b200.unet import CrossAttention, UNetConfig, attention_modules, build_unet
from tests.fixtures import SETTINGS, color_map_image
from tests.golden.make_long_prompt_golden import LONG_AURORA_PROMPT
from tests.test_xattn_gpu import IMPLS, RAGGED, SD15_256, SD15_512, SD21_768, _inputs, _oracle, _run

pytestmark = pytest.mark.gpu
LONG_T = [154, 231]


@pytest.mark.parametrize("impl", IMPLS)
@pytest.mark.parametrize("N,H,D", SD15_512 + SD15_256 + SD21_768 + RAGGED)
@pytest.mark.parametrize("stat", ["max", "std"])
@pytest.mark.parametrize("T", LONG_T)
def test_long_bias_path_matches_oracle(T, N, H, D, stat, impl):
    if stat == "std" and N * H > 40000:
        pytest.skip("std covered at the smaller sizes; max covers the large ones")
    q, k, v, w = _inputs(1, N, H, D, T, seed=N * 131 + D + T)
    scale = D ** -0.5
    g = 0.4 * math.log(1 + 7.0) if stat == "max" else 0.5 * math.log(1 + 7.0 ** 2)
    got, st = _run(q, k, v, H, scale, w, g, stat, impl=impl)
    ref16, st16 = _oracle(q, k, v, H, scale, w, g, stat, emulate=True)
    ref32, _ = _oracle(q, k, v, H, scale, w, g, stat, emulate=False)
    assert abs(float(st[0]) - st16[0]) <= 2 ** -10 * abs(st16[0]) + 1e-6, (float(st[0]), st16[0])
    amax = ref32.abs().max().item()
    assert (got - ref16).abs().max().item() <= 1.5e-3 * amax
    assert (got - ref32).abs().max().item() <= 2e-3 * amax


@pytest.mark.parametrize("impl", IMPLS)
@pytest.mark.parametrize("N,H,D", [(4096, 8, 40), (64, 8, 160), (576, 20, 64), (1024, 8, 80)])
def test_long_plain_cross_attention_matches_oracle(N, H, D, impl):
    q, k, v, _ = _inputs(2, N, H, D, 154, seed=17)
    got, st = _run(q, k, v, H, D ** -0.5, None, 0.0, "max", impl=impl)
    ref32, _ = _oracle(q, k, v, H, D ** -0.5, None, 0.0, "max", emulate=False)
    assert st is None
    assert (got - ref32).abs().max().item() <= 2e-3 * ref32.abs().max().item()


@pytest.mark.parametrize("impl", IMPLS)
@pytest.mark.parametrize("T", LONG_T)
def test_long_batched_cfg_per_image_stats(T, impl):
    """[cond0, uncond, cond1] in one call at a long context; batching does not change an image's result."""
    N, H, D = 1024, 8, 80
    q, k, v, w = _inputs(3, N, H, D, T, seed=99 + T)
    q[2] *= 3.0
    idx = torch.tensor([1, -1, 0], dtype=torch.int32)
    g = 0.4 * math.log(1 + 3.0)
    got, st = _run(q, k, v, H, D ** -0.5, w[:2].contiguous(), g, "max", idx, impl=impl)
    w_eff = torch.stack([w[1], torch.zeros_like(w[0]), w[0]])
    ref, stats = _oracle(q, k, v, H, D ** -0.5, w_eff, g, "max", emulate=False)
    ref_plain, _ = _oracle(q[1:2], k[1:2], v[1:2], H, D ** -0.5, None, 0.0, "max", emulate=False)
    amax = ref.abs().max().item()
    assert (got[0] - ref[0]).abs().max().item() <= 2e-3 * amax
    assert (got[2] - ref[2]).abs().max().item() <= 2e-3 * amax
    assert (got[1] - ref_plain[0]).abs().max().item() <= 2e-3 * amax
    assert float(st[1]) == 0.0 and abs(float(st[2]) - stats[2]) <= 2e-3 * abs(stats[2])
    solo, st_solo = _run(q[2:3], k[2:3], v[2:3], H, D ** -0.5, w[0:1].contiguous(), g, "max", impl=impl)
    assert torch.equal(solo[0], got[2]) and float(st_solo[0]) == float(st[2])


@pytest.mark.parametrize("T", LONG_T)
def test_long_launch_counts(T):
    """A packable map is one native launch; a map with 11 distinct columns takes the dense pair (two launches)."""
    N, H, D = 1024, 8, 40
    q, k, v, w = _inputs(1, N, H, D, T, seed=T + 5)
    before = _native.launch_count
    got, _ = _run(q, k, v, H, D ** -0.5, w, 0.6, "max", impl="auto")
    assert _native.launch_count - before == 1
    ref32, _ = _oracle(q, k, v, H, D ** -0.5, w, 0.6, "max", emulate=False)
    assert (got - ref32).abs().max().item() <= 2e-3 * ref32.abs().max().item()
    gen = torch.Generator().manual_seed(T)
    w11 = torch.zeros(1, N, T)
    for j, t in enumerate(torch.randperm(T, generator=gen)[:11]):       # 11 regions spread over the chunks
        w11[0, :, t] = (torch.rand(N, generator=gen) > 0.5).float() * (0.5 + 0.1 * j)
    assert C.pack_weight_map(w11) is None
    before = _native.launch_count
    got, _ = _run(q, k, v, H, D ** -0.5, w11, 0.6, "max", impl="auto")
    assert _native.launch_count - before == 2
    ref32, _ = _oracle(q, k, v, H, D ** -0.5, w11, 0.6, "max", emulate=False)
    assert (got - ref32).abs().max().item() <= 2e-3 * ref32.abs().max().item()


@torch.no_grad()
def test_long_inj_forward_dict_and_orig_fallback():
    """inj_forward with a 154-token dict context: a weight map of this level, then only the ORIG map (expanded by the
    reference's KeyError path)."""
    g = torch.Generator().manual_seed(3)
    heads, d, N, dc, T = 2, 40, 64, 32, 154
    attn = CrossAttention(heads * d, dc, heads, d)
    for p in attn.parameters():
        p.data = torch.randn(p.shape, generator=g) * (0.3 if p.dim() > 1 else 0.05)
    x = torch.randn(1, N, heads * d, generator=g)
    ctx = torch.randn(1, T, dc, generator=g)
    w_orig = torch.zeros(24, 24, T)
    w_orig[4:14, 6:20, 5] = 2.0
    w_orig[10:24, 0:9, 100:102] = 0.7
    f = lambda w, sigma, qk: 0.4 * w * math.log(1 + sigma) * qk.max()   # noqa: E731
    sigma = torch.tensor(7.25)
    w = C.expand_orig_weight_map(w_orig, N)
    attn_d = CrossAttention(heads * d, dc, heads, d).cuda()
    attn_d.load_state_dict(attn.state_dict())
    for c in ({"CONTEXT_TENSOR": ctx, f"CROSS_ATTENTION_WEIGHT_{N}": w, "CROSS_ATTENTION_WEIGHT_ORIG": 0},
              {"CONTEXT_TENSOR": ctx, "CROSS_ATTENTION_WEIGHT_ORIG": w_orig}):
        c = dict(c, SIGMA=sigma, WEIGHT_FUNCTION=f)
        ref = O.inj_forward(attn, x, dict(c))
        cd = {k_: (v_.cuda() if isinstance(v_, torch.Tensor) and k_ != "CROSS_ATTENTION_WEIGHT_ORIG" else v_)
              for k_, v_ in c.items()}
        got = A.inj_forward(attn_d, x.cuda(), cd).float().cpu()
        assert (got - ref).abs().max().item() <= 2e-3 * ref.abs().max().item()


WF = lambda w, sigma, qk: 0.4 * w * math.log(1 + sigma) * qk.max()   # noqa: E731


def _setup(cfg, size, steps, device):
    tok, enc = SimpleWordTokenizer(), RandomTextEncoder(cfg.cross_attention_dim)
    s = SETTINGS["aurora"]
    _, _, cond, uncond = C._encode_text_color_inputs(enc.to(device), tok, device, color_map_image("aurora", size),
                                                     dict(s["ctx"]), LONG_AURORA_PROMPT, "", max_prompt_chunks=3)
    sch = LMSDiscreteScheduler(beta_start=0.00085, beta_end=0.012, beta_schedule="scaled_linear")
    sch.set_timesteps(steps)
    lat = torch.randn(1, 4, size // 8, size // 8, generator=torch.manual_seed(0)) * sch.init_noise_sigma
    return cond, uncond, sch, lat


@pytest.mark.parametrize("use_graph", [False, True])
def test_sampler_with_two_chunk_prompt_matches_reference_loop(use_graph):
    cfg = UNetConfig.tiny()
    size, steps = 128, 4
    unet = build_unet(cfg, seed=0)
    cond, uncond, sch, lat = _setup(cfg, size, steps, "cpu")
    assert cond["CONTEXT_TENSOR"].shape[1] == 154 and uncond["CONTEXT_TENSOR"].shape[1] == 154
    try:
        oracle_loop.patch_with_oracle(unet)
        ref = oracle_loop.reference_denoise_loop(unet, sch, cond, uncond, lat, WF)
    finally:
        cls = attention_modules(unet)[0].__class__
        if "__call__" in cls.__dict__:
            delattr(cls, "__call__")
    unet = build_unet(cfg, seed=0, dtype=torch.float16, device="cuda")
    cond, uncond, sch, lat = _setup(cfg, size, steps, "cuda")
    try:
        P.patch_unet(unet)
        out = PwWSampler(unet, sch, [cond], [uncond], lat.cuda(), WF, 7.5, use_graph=use_graph).run()
    finally:
        P.unpatch_all()
    out = out.float().cpu()
    rel_rmse = ((out - ref).pow(2).mean().sqrt() / ref.pow(2).mean().sqrt()).item()
    assert torch.isfinite(out).all() and rel_rmse < 3e-2, rel_rmse


def test_sampler_rejects_mixed_text_lengths():
    cfg = UNetConfig.tiny()
    unet = build_unet(cfg, seed=0, dtype=torch.float16, device="cuda")
    long_c, long_u, sch, lat = _setup(cfg, 128, 2, "cuda")
    tok, enc = SimpleWordTokenizer(), RandomTextEncoder(cfg.cross_attention_dim).cuda()
    s = SETTINGS["aurora"]
    _, _, short_c, short_u = C._encode_text_color_inputs(enc, tok, "cuda", color_map_image("aurora", 128),
                                                         dict(s["ctx"]), s["prompt"], "")
    with pytest.raises(ValueError):
        PwWSampler(unet, sch, [long_c, short_c], [long_u, short_u], torch.cat([lat, lat]).cuda(), WF, 7.5)
