"""Region prompts on the GPU: the region kernel through the C ABI against the fp32 oracle (oracle/region_prompt.py),
equivalences that must hold exactly in exact arithmetic, loop parity against the oracle loop, and the step's launch
count.  Tolerances are test_xattn_gpu.py's for the streaming kernel: 2e-3 * max|out| against the fp32 oracle in fp16,
1.6e-2 in bf16 (test_bf16_gpu.py); loops: relative RMSE < 3e-2."""
import math

import pytest
import torch

import paint_with_words_sd_b200 as P
from oracle import controlnet_loop
from oracle import region_prompt as RO
from paint_with_words_sd_b200 import _native
from paint_with_words_sd_b200 import attention as A
from paint_with_words_sd_b200 import conditioning as C
from paint_with_words_sd_b200.controlnet import build_controlnet
from paint_with_words_sd_b200.pipeline import PwWSampler
from paint_with_words_sd_b200.scheduler import DPMSolverMultistepScheduler, LMSDiscreteScheduler
from paint_with_words_sd_b200.synthetic import RandomTextEncoder, SimpleWordTokenizer
from paint_with_words_sd_b200.unet import UNetConfig, attention_modules, build_unet
from tests.fixtures import SETTINGS, color_map_image
from tests.test_xattn_gpu import RAGGED, SD15_256, SD15_512, SD21_768

pytestmark = pytest.mark.gpu
TOL = {torch.float16: 2e-3, torch.bfloat16: 1.6e-2}


def _weights(B, N, kc, g):
    """Convex rows with exact 0 / 1 entries on some rows, and chunk kc - 1 unweighted on the whole first row tile."""
    w = torch.rand(B, N, kc, generator=g)
    w[:, : min(N, 128), kc - 1] = 0.0
    w = w / w.sum(-1, keepdim=True)
    for b in range(B):
        rows = torch.randperm(N, generator=g)[: max(1, N // 7)]
        one_hot = torch.randint(0, kc, (len(rows),), generator=g)
        w[b, rows] = torch.nn.functional.one_hot(one_hot, kc).float()
    return w.contiguous()


def _case(B, N, H, D, kc, dtype, seed):
    g = torch.Generator().manual_seed(seed)
    T, Cc = 77 * kc, H * D
    q = (torch.randn(B, N, Cc, generator=g) * 0.5).to(dtype)
    k = (torch.randn(B, T, Cc, generator=g) * 0.5).to(dtype)
    v = (torch.randn(B, T, Cc, generator=g) * 0.5).to(dtype)
    wmap = torch.zeros(B, N, T)
    for b in range(B):
        for c in torch.randperm(T, generator=g)[:9]:
            wmap[b, :, c] += (torch.rand(N, generator=g) > 0.6).float() * float(torch.rand(1, generator=g) * 2)
    return q, k, v, wmap, _weights(B, N, kc, g)


def _oracle(q, k, v, H, scale, wmap, rw, g, stats):
    outs, st = [], []
    for b in range(q.shape[0]):
        box = {}

        def bias(s, b=b):
            m = s.max() if stats[b] == "max" else s.std()
            box["m"] = float(m)
            return g[b] * wmap[b] * m
        outs.append(RO.region_attention_core(q[b:b + 1].float(), k[b:b + 1].float(), v[b:b + 1].float(), H, scale,
                                             None if rw is None or rw[b] is None else rw[b],
                                             bias if g[b] is not None else None))
        st.append(box.get("m"))
    return torch.cat(outs, 0), st


@pytest.mark.parametrize("mode", ["plain", "biased", "biased_multi"])
@pytest.mark.parametrize("stat", ["max", "std"])
@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16], ids=["f16", "bf16"])
@pytest.mark.parametrize("kc", [2, 3])
@pytest.mark.parametrize("N,H,D", SD15_512 + SD15_256 + SD21_768 + RAGGED)
def test_region_kernel_matches_oracle(N, H, D, kc, dtype, stat, mode):
    if mode == "plain" and stat == "std":
        pytest.skip("no statistic without a bias")
    if stat == "std" and N * H > 40000:
        pytest.skip("std covered at the smaller sizes; max covers the large ones")
    B = 3                                                  # cond, uncond (no weights: first chunk alone), cond
    q, k, v, wmap, rw = _case(B, N, H, D, kc, dtype, seed=N * 7 + D + kc)
    scale = D ** -0.5
    idx = torch.tensor([0, -1, 1], dtype=torch.int32)
    stats = [stat, stat, "std" if mode == "biased_multi" else stat]
    gs = [0.4 * math.log(8.0), None, 0.3 * math.log(8.0)]
    if mode != "biased_multi":
        gs[2] = gs[0]
    dev = "cuda"
    region = rw[[0, 2]].to(dev)
    if mode == "plain":
        out = A.cross_attention(q.to(dev), k.to(dev), v.to(dev), H, scale, wmap_index=idx.to(dev), region=region)
        ref, _ = _oracle(q, k, v, H, scale, None, [rw[0], None, rw[2]], [None] * 3, stats)
        st = None
    else:
        kinds = torch.tensor([_native.PWW_STAT_MAX if s == "max" else _native.PWW_STAT_STD for s in stats],
                             dtype=torch.int32, device=dev)
        if mode == "biased_multi":
            stat_arg, g_dev = kinds, torch.tensor([gs[0], 0.0, gs[2]], dtype=torch.float32, device=dev)
        else:
            stat_arg, g_dev = int(kinds[0]), torch.tensor([gs[0]], dtype=torch.float32, device=dev)
        before = _native.launch_count
        out, st = A.cross_attention(q.to(dev), k.to(dev), v.to(dev), H, scale, wmap[[0, 2]].to(dev), idx.to(dev),
                                    stat_arg, g_dev, return_stats=True, region=region)
        assert _native.launch_count - before == 1
        ref, ref_st = _oracle(q, k, v, H, scale, [wmap[0], None, wmap[2]], [rw[0], None, rw[2]], gs, stats)
        st = st.cpu()
        for b in (0, 2):
            rel = 2e-3 if dtype == torch.float16 else 2 ** -8     # the statistic is rounded to E
            assert abs(float(st[b]) - ref_st[b]) <= rel * abs(ref_st[b]) + 1e-6, (b, float(st[b]), ref_st[b])
    out = out.float().cpu()
    assert torch.isfinite(out).all()
    amax = ref.abs().max().item()
    err = (out - ref).abs().max().item()
    assert err <= TOL[dtype] * amax, (err / amax)


def test_chunks_no_row_weighs_are_not_read():
    """Every row weighs chunk 1 alone: chunks 0 and 2 are never read, so poisoning their V changes no bit."""
    N, H, D = 256, 8, 40
    q, k, v, _, _ = _case(1, N, H, D, 3, torch.float16, seed=5)
    w = torch.zeros(1, N, 3)
    w[..., 1] = 1.0
    dev = "cuda"
    a = A.cross_attention(q.to(dev), k.to(dev), v.to(dev), H, D ** -0.5, region=w.to(dev))
    v2 = v.clone()
    v2[:, :77] = 3.0e4
    v2[:, 154:] = float("inf")
    b = A.cross_attention(q.to(dev), k.to(dev), v2.to(dev), H, D ** -0.5, region=w.to(dev))
    assert torch.equal(a, b)


# ---------------------------------------------------------------------------------------------------------------
# the sampler
# ---------------------------------------------------------------------------------------------------------------
SIZE = 128
WF = lambda w, sigma, qk: 0.4 * w * math.log(1 + sigma) * qk.max()   # noqa: E731
WF_ZERO = lambda w, sigma, qk: 0.0 * w                                # noqa: E731


def _regions(name):
    ctx = SETTINGS[name]["ctx"]
    colours = list(ctx)
    return {colours[0]: "a small red lantern glowing", colours[-1]: "a tall green tree"}


def _encode(device, name="cat_dog", region_prompts=None, beta=0.2, cfg=None):
    cfg = cfg or UNetConfig.tiny()
    tok, enc = SimpleWordTokenizer(), RandomTextEncoder(cfg.cross_attention_dim).to(device)
    s = SETTINGS[name]
    _, _, cond, uncond = C._encode_text_color_inputs(enc, tok, device, color_map_image(name, SIZE), dict(s["ctx"]),
                                                     s["prompt"], "", region_prompts=region_prompts,
                                                     region_base_ratio=beta)
    return cond, uncond


def _sch(cls=LMSDiscreteScheduler, steps=4):
    sch = cls(beta_start=0.00085, beta_end=0.012, beta_schedule="scaled_linear")
    sch.set_timesteps(steps)
    return sch


def _lat(seed, sch):
    return torch.randn(1, 4, SIZE // 8, SIZE // 8, generator=torch.manual_seed(seed)) * sch.init_noise_sigma


def _run_gpu(conds, unconds, lats, wf, sch, dtype=torch.float16, use_graph=True, **kw):
    unet = build_unet(UNetConfig.tiny(), seed=0, dtype=dtype, device="cuda")
    P.patch_unet(unet)
    try:
        s = PwWSampler(unet, sch, conds, unconds, torch.cat(lats, 0).cuda(), wf, 7.5, use_graph=use_graph, **kw)
        return s.run().float().cpu(), s
    finally:
        P.unpatch_all()


def _rel_rmse(a, b):
    return ((a - b).pow(2).mean().sqrt() / b.pow(2).mean().sqrt()).item()


def _unpatch(unet):
    cls = attention_modules(unet)[0].__class__
    if "__call__" in cls.__dict__:
        delattr(cls, "__call__")


@pytest.mark.parametrize("case", ["beta_one", "absent_colour"])
def test_region_prompts_that_weigh_nothing_equal_the_plain_call(case):
    """Without a bias (the statistic spans every chunk, so a biased call differs by design): beta = 1, or a region
    colour that the map does not contain, leaves the base prompt alone on every pixel."""
    regions = {(1, 2, 3): "a tall green tree"} if case == "absent_colour" else _regions("cat_dog")
    beta = 1.0 if case == "beta_one" else 0.2
    sch = _sch()
    cond, uncond = _encode("cuda", region_prompts=regions, beta=beta)
    got, _ = _run_gpu([cond], [uncond], [_lat(0, sch)], WF_ZERO, sch)
    sch = _sch()
    cond, uncond = _encode("cuda")
    ref, _ = _run_gpu([cond], [uncond], [_lat(0, sch)], WF_ZERO, sch)
    assert _rel_rmse(got, ref) < 1e-2


def test_batch_of_region_images_equals_each_alone():
    sch = _sch()
    a = _encode("cuda", "cat_dog", _regions("cat_dog"))
    b = _encode("cuda", "aurora", _regions("aurora"), beta=0.5)
    both, _ = _run_gpu([a[0], b[0]], [a[1], b[1]], [_lat(0, sch), _lat(1, sch)], [WF, WF_ZERO], sch)
    for i, (c, u) in enumerate((a, b)):
        alone, _ = _run_gpu([c], [u], [_lat(i, sch)], [WF, WF_ZERO][i], _sch())
        assert (both[i:i + 1] - alone).abs().max().item() <= 2e-2 * alone.abs().max().item()


def test_public_batch_of_a_region_image_and_a_plain_image_equals_each_alone():
    from paint_with_words_sd_b200.synthetic import IdentityVAE
    cfg = UNetConfig.tiny()
    unet = build_unet(cfg, seed=0, dtype=torch.float16, device="cuda")
    tools = (IdentityVAE(), unet, RandomTextEncoder(cfg.cross_attention_dim).cuda(), SimpleWordTokenizer(),
             LMSDiscreteScheduler(beta_start=0.00085, beta_end=0.012, beta_schedule="scaled_linear"))
    s = SETTINGS["cat_dog"]
    base = dict(color_context=dict(s["ctx"]), color_map_image=color_map_image("cat_dog", SIZE),
                input_prompt=s["prompt"])
    entries = [dict(base, seed=0, region_prompts=_regions("cat_dog")), dict(base, seed=1)]
    P.patch_unet(unet)
    try:
        both = P.paint_with_words_batch(entries, num_inference_steps=3, device="cuda", preloaded_utils=tools,
                                        return_latents=True)
        alone = [P.paint_with_words(**e, num_inference_steps=3, device="cuda", preloaded_utils=tools,
                                    return_latents=True) for e in entries]
    finally:
        P.unpatch_all()
    for x, y in zip(both, alone):
        assert (x - y).abs().max().item() <= 2e-2 * y.abs().max().item()


def test_sampler_with_region_prompts_matches_oracle_loop_lms():
    cfg = UNetConfig.tiny()
    unet = build_unet(cfg, seed=0)
    regions = _regions("cat_dog")
    sch = _sch()
    cond, uncond = _encode("cpu", region_prompts=regions)
    try:
        RO.patch_with_region_oracle(unet)
        ref = RO.reference_region_loop(unet, sch, cond, uncond, _lat(0, sch), WF)
    finally:
        _unpatch(unet)
    sch = _sch()
    cond, uncond = _encode("cuda", region_prompts=regions)
    out, _ = _run_gpu([cond], [uncond], [_lat(0, sch)], WF, sch)
    assert torch.isfinite(out).all() and _rel_rmse(out, ref) < 3e-2, _rel_rmse(out, ref)


def test_sampler_with_region_prompts_matches_oracle_loop_dpm_controlnet():
    from tests.test_controlnet_gpu import _hint
    cfg = UNetConfig.tiny()
    unet, net = build_unet(cfg, seed=0), build_controlnet(UNetConfig.tiny(), seed=1)
    regions = _regions("aurora")
    sch = _sch(DPMSolverMultistepScheduler)
    cond, uncond = _encode("cpu", "aurora", regions)
    try:
        RO.patch_with_region_oracle(unet)
        ref = controlnet_loop.reference_controlnet_loop(unet, net, sch, cond, uncond, _lat(0, sch), WF, _hint(0), 7.5,
                                                        0.8)
    finally:
        _unpatch(unet)
    sch = _sch(DPMSolverMultistepScheduler)
    cond, uncond = _encode("cuda", "aurora", regions)
    net = build_controlnet(UNetConfig.tiny(), seed=1, dtype=torch.float16, device="cuda")
    out, _ = _run_gpu([cond], [uncond], [_lat(0, sch)], WF, sch, controlnet=net, control_image=_hint(0),
                      controlnet_conditioning_scale=0.8)
    assert torch.isfinite(out).all() and _rel_rmse(out, ref) < 3e-2, _rel_rmse(out, ref)


@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16], ids=["f16", "bf16"])
def test_region_step_has_as_many_launches_as_a_plain_step_and_replays(dtype):
    sch = _sch()
    cond, uncond = _encode("cuda", region_prompts=_regions("cat_dog"))
    graph, s = _run_gpu([cond], [uncond], [_lat(0, sch)], WF, sch, dtype=dtype)
    eager, _ = _run_gpu([cond], [uncond], [_lat(0, sch)], WF, _sch(), dtype=dtype, use_graph=False)
    sch = _sch()
    pc, pu = _encode("cuda")
    _, plain = _run_gpu([pc], [pu], [_lat(0, sch)], WF, sch, dtype=dtype)
    assert s.native_launches_per_step is not None
    assert s.native_launches_per_step == plain.native_launches_per_step
    assert torch.isfinite(graph).all()
    assert (graph - eager).abs().max().item() <= 1e-3 * eager.abs().max().item()
