"""Negative region prompts on the GPU: `pww_xattn_fused_region_rows_*` through the C ABI against the fp32 oracle
(oracle/negative_region.py) for batches that mix every kind of row, its bits against `pww_xattn_fused_region_*`,
chunks it must not read, sampler parity against the oracle loop, exact equivalences, the public batch and the step's
launch count.  Tolerances are test_region_prompts_gpu.py's."""
import math

import pytest
import torch

import paint_with_words_sd_b200 as P
from oracle import controlnet_loop
from oracle import negative_region as NO
from oracle import region_prompt as RO
from paint_with_words_sd_b200 import _native
from paint_with_words_sd_b200 import attention as A
from paint_with_words_sd_b200 import conditioning as C
from paint_with_words_sd_b200.controlnet import build_controlnet
from paint_with_words_sd_b200.pipeline import PwWSampler
from paint_with_words_sd_b200.scheduler import DPMSolverMultistepScheduler, LMSDiscreteScheduler
from paint_with_words_sd_b200.synthetic import IdentityVAE, RandomTextEncoder, SimpleWordTokenizer
from paint_with_words_sd_b200.unet import UNetConfig, build_unet
from tests.fixtures import SETTINGS, color_map_image
from tests.test_region_prompts_gpu import (SIZE, WF, WF_ZERO, _case, _lat, _rel_rmse, _run_gpu, _sch, _unpatch,
                                           _weights)

pytestmark = pytest.mark.gpu
TOL = {torch.float16: 2e-3, torch.bfloat16: 1.6e-2}
SHAPES = [(4096, 8, 40), (1024, 8, 80), (256, 8, 160), (64, 8, 160), (2304, 10, 64), (333, 1, 160), (129, 3, 80)]
ABSENT = (1, 2, 3)


def _rows_case(N, H, D, kc, dtype, seed):
    """Five images: biased with weights and every chunk in its statistic; biased with row -1 and statistic {0}; biased
    with weights and a partial statistic; unbiased with weights; unbiased with row -1."""
    q, k, v, wmap, _ = _case(5, N, H, D, kc, dtype, seed)
    g = torch.Generator().manual_seed(seed + 1)
    rw = _weights(3, N, kc, g)
    wmap_index = torch.tensor([0, 1, 2, -1, -1], dtype=torch.int32)
    region_index = torch.tensor([0, -1, 1, 2, -1], dtype=torch.int32)
    full = (1 << kc) - 1
    stat_chunks = torch.tensor([full, 1, 0b101 if kc == 3 else 0b01, full, full], dtype=torch.int32)
    return q, k, v, wmap[:3].contiguous(), rw, wmap_index, region_index, stat_chunks


def _oracle(q, k, v, H, scale, wmap, wmap_index, rw, region_index, masks, gs, stats):
    outs, st = [], []
    T = k.shape[1]
    for b in range(q.shape[0]):
        box = {}
        cols = NO.stat_columns(int(masks[b]), T)

        def bias(s, b=b, cols=cols):
            sub = s[..., cols]
            m = sub.max() if stats[b] == "max" else sub.std()
            box["m"] = float(m)
            return gs[b] * wmap[int(wmap_index[b])] * m
        ri = int(region_index[b])
        outs.append(RO.region_attention_core(q[b:b + 1].float(), k[b:b + 1].float(), v[b:b + 1].float(), H, scale,
                                             rw[ri] if ri >= 0 else None,
                                             bias if int(wmap_index[b]) >= 0 else None))
        st.append(box.get("m"))
    return torch.cat(outs, 0), st


def _call(q, k, v, H, scale, wmap, wmap_index, rw, rows, stat, g_dev, dev="cuda"):
    return A.cross_attention(q.to(dev), k.to(dev), v.to(dev), H, scale, wmap.to(dev), wmap_index.to(dev), stat, g_dev,
                             return_stats=True, region=rw.to(dev), region_rows=rows)


@pytest.mark.parametrize("multi", [False, True], ids=["single", "multi"])
@pytest.mark.parametrize("stat", ["max", "std"])
@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16], ids=["f16", "bf16"])
@pytest.mark.parametrize("kc", [2, 3])
@pytest.mark.parametrize("N,H,D", SHAPES)
def test_region_rows_kernel_matches_oracle(N, H, D, kc, dtype, stat, multi):
    q, k, v, wmap, rw, widx, ridx, masks = _rows_case(N, H, D, kc, dtype, seed=N * 3 + D + kc)
    scale = D ** -0.5
    dev = "cuda"
    gs = [0.4 * math.log(8.0)] * 3 + [None, None]
    stats = [stat] * 5
    if multi:
        gs[1], stats[2] = 0.3 * math.log(8.0), ("std" if stat == "max" else "max")
        kinds = torch.tensor([_native.PWW_STAT_MAX if s == "max" else _native.PWW_STAT_STD for s in stats],
                             dtype=torch.int32, device=dev)
        stat_arg = kinds
        g_dev = torch.tensor([g or 0.0 for g in gs], dtype=torch.float32, device=dev)
    else:
        stat_arg = _native.PWW_STAT_MAX if stat == "max" else _native.PWW_STAT_STD
        g_dev = torch.tensor([gs[0]], dtype=torch.float32, device=dev)
    before = _native.launch_count
    out, st = _call(q, k, v, H, scale, wmap, widx, rw, (ridx.to(dev), masks.to(dev)), stat_arg, g_dev)
    assert _native.launch_count - before == 1
    ref, ref_st = _oracle(q, k, v, H, scale, wmap, widx, rw, ridx, masks, gs, stats)
    st = st.cpu()
    for b in range(3):
        rel = 2e-3 if dtype == torch.float16 else 2 ** -8          # the statistic is rounded to E
        assert abs(float(st[b]) - ref_st[b]) <= rel * abs(ref_st[b]) + 1e-6, (b, float(st[b]), ref_st[b])
    out = out.float().cpu()
    assert torch.isfinite(out).all()
    amax = ref.abs().max().item()
    for b in range(5):
        err = (out[b] - ref[b]).abs().max().item()
        assert err <= TOL[dtype] * amax, (b, err / amax)


@pytest.mark.parametrize("biased", [False, True])
@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16], ids=["f16", "bf16"])
@pytest.mark.parametrize("kc", [2, 3])
@pytest.mark.parametrize("N,H,D", [(4096, 8, 40), (1024, 8, 80), (333, 1, 160)])
def test_region_rows_with_the_bias_index_give_the_region_entry_points_bits(N, H, D, kc, dtype, biased):
    q, k, v, wmap, rw, _, _, _ = _rows_case(N, H, D, kc, dtype, seed=N + D + kc)
    idx = torch.tensor([0, -1, 2, -1, 1], dtype=torch.int32, device="cuda")
    g_dev = torch.tensor([0.5], dtype=torch.float32, device="cuda")
    kw = dict(region=rw.cuda())
    if biased:
        kw.update(wmap=wmap.cuda(), wmap_index=idx, stat=_native.PWW_STAT_STD, g_sigma=g_dev, return_stats=True)
    else:
        kw.update(wmap_index=idx)
    args = (q.cuda(), k.cuda(), v.cuda(), H, D ** -0.5)
    a = A.cross_attention(*args, **kw)
    b = A.cross_attention(*args, **kw, region_rows=(idx, None))
    if biased:
        assert torch.equal(a[1], b[1])
        a, b = a[0], b[0]
    assert torch.equal(a, b)


@pytest.mark.parametrize("kc", [2, 3])
def test_chunks_outside_an_images_statistic_and_weights_are_not_read(kc):
    N, H, D = 1024, 8, 80
    q, k, v, wmap, _, _, _, _ = _rows_case(N, H, D, kc, torch.float16, seed=7)
    q, k, v = q[:3], k[:3], v[:3]
    rw = torch.zeros(2, N, kc)
    rw[0, :, 0], rw[0, :, 1] = 0.3, 0.7                    # image 0: chunks 0 and 1
    rw[1, :, 0] = 1.0
    widx = torch.tensor([0, 1, -1], dtype=torch.int32, device="cuda")
    ridx = torch.tensor([0, -1, -1], dtype=torch.int32, device="cuda")
    masks = torch.tensor([0b011, 1, 1], dtype=torch.int32, device="cuda")
    g_dev = torch.tensor([0.4 * math.log(8.0)], dtype=torch.float32, device="cuda")

    def run(k, v):
        return A.cross_attention(q.cuda(), k.cuda(), v.cuda(), H, D ** -0.5, wmap[:2].cuda(), widx,
                                 _native.PWW_STAT_MAX, g_dev, return_stats=True, region=rw.cuda(),
                                 region_rows=(ridx, masks))
    a, sa = run(k, v)
    k2, v2 = k.clone(), v.clone()
    k2[1:, 77:], v2[1:, 77:] = float("nan"), float("nan")             # images 1, 2: every chunk but 0
    if kc == 3:
        k2[0, 154:], v2[0, 154:] = float("nan"), float("nan")         # image 0: chunk 2
    b, sb = run(k2, v2)
    assert torch.isfinite(a).all()
    assert torch.equal(a, b) and torch.equal(sa[:2], sb[:2])


# ---------------------------------------------------------------------------------------------------------------
# the sampler
# ---------------------------------------------------------------------------------------------------------------
def _colours(name="cat_dog"):
    return list(SETTINGS[name]["ctx"])


def _encode(device, name="cat_dog", region_prompts=None, negative=None, beta=0.2, uncond="blurry", cfg=None):
    cfg = cfg or UNetConfig.tiny()
    tok, enc = SimpleWordTokenizer(), RandomTextEncoder(cfg.cross_attention_dim).to(device)
    s = SETTINGS[name]
    _, _, cond, uncond = C._encode_text_color_inputs(enc, tok, device, color_map_image(name, SIZE), dict(s["ctx"]),
                                                     s["prompt"], uncond, region_prompts=region_prompts,
                                                     region_base_ratio=beta, negative_region_prompts=negative)
    return cond, uncond


def _mixed(name="cat_dog"):
    c = _colours(name)
    return {c[0]: "a small red lantern glowing"}, {c[-1]: "tall green trees"}


def _oracle_loop(name, pos, neg, sch, controlnet=None):
    unet = build_unet(UNetConfig.tiny(), seed=0)
    cond, uncond = _encode("cpu", name, pos, neg)
    try:
        NO.patch_with_negative_region_oracle(unet)
        if controlnet is None:
            return RO.reference_region_loop(unet, sch, cond, uncond, _lat(0, sch), WF)
        from tests.test_controlnet_gpu import _hint
        return controlnet_loop.reference_controlnet_loop(unet, controlnet, sch, cond, uncond, _lat(0, sch), WF,
                                                         _hint(0), 7.5, 0.8)
    finally:
        _unpatch(unet)


@pytest.mark.parametrize("case", ["mixed", "negative_only"])
def test_sampler_with_negative_regions_matches_oracle_loop_lms(case):
    pos, neg = _mixed()
    if case == "negative_only":
        pos = None
    ref = _oracle_loop("cat_dog", pos, neg, _sch())
    sch = _sch()
    cond, uncond = _encode("cuda", "cat_dog", pos, neg)
    out, _ = _run_gpu([cond], [uncond], [_lat(0, sch)], WF, sch)
    assert torch.isfinite(out).all() and _rel_rmse(out, ref) < 3e-2, _rel_rmse(out, ref)


def test_sampler_with_negative_regions_matches_oracle_loop_dpm_controlnet():
    from tests.test_controlnet_gpu import _hint
    pos, neg = _mixed("aurora")
    ref = _oracle_loop("aurora", pos, neg, _sch(DPMSolverMultistepScheduler),
                       controlnet=build_controlnet(UNetConfig.tiny(), seed=1))
    sch = _sch(DPMSolverMultistepScheduler)
    cond, uncond = _encode("cuda", "aurora", pos, neg)
    net = build_controlnet(UNetConfig.tiny(), seed=1, dtype=torch.float16, device="cuda")
    out, _ = _run_gpu([cond], [uncond], [_lat(0, sch)], WF, sch, controlnet=net, control_image=_hint(0),
                      controlnet_conditioning_scale=0.8)
    assert torch.isfinite(out).all() and _rel_rmse(out, ref) < 3e-2, _rel_rmse(out, ref)


@pytest.mark.parametrize("case", ["absent_colour", "beta_one"])
def test_negative_regions_that_weigh_nothing_give_the_same_bits(case):
    """The uncond rows then weigh chunk 0 alone, exactly as without negatives, and the cond side is unchanged."""
    c = _colours()
    if case == "absent_colour":
        pos, neg, beta = {c[0]: "a small red lantern", ABSENT: "a tall tree"}, {ABSENT: "green trees"}, 0.2
    else:
        pos, neg, beta = {c[0]: "a small red lantern", c[-1]: "a tall tree"}, {c[-1]: "green trees"}, 1.0
    sch = _sch()
    cond, uncond = _encode("cuda", region_prompts=pos, negative=neg, beta=beta)
    got, _ = _run_gpu([cond], [uncond], [_lat(0, sch)], WF, sch)
    sch = _sch()
    cond, uncond = _encode("cuda", region_prompts=pos, beta=beta)
    ref, _ = _run_gpu([cond], [uncond], [_lat(0, sch)], WF, sch)
    assert torch.equal(got, ref)


def test_negative_only_cond_half_is_the_plain_calls():
    """Guidance scale 1 keeps the cond half alone: its bias statistic is chunk 0's, the plain call's 77 keys."""
    _, neg = _mixed()
    cond, uncond = _encode("cuda", negative=neg)
    assert cond[C.REGION_SENTENCES_KEY] == 0
    unet = build_unet(UNetConfig.tiny(), seed=0, dtype=torch.float16, device="cuda")
    P.patch_unet(unet)
    try:
        outs = []
        for c, u in ((cond, uncond), _encode("cuda")):
            sch = _sch()
            outs.append(PwWSampler(unet, sch, [c], [u], _lat(0, sch).cuda(), WF, 1.0).run().float().cpu())
    finally:
        P.unpatch_all()
    assert torch.isfinite(outs[0]).all()
    assert _rel_rmse(outs[0], outs[1]) < 1e-2, _rel_rmse(outs[0], outs[1])


def test_public_batch_of_every_kind_equals_each_alone():
    cfg = UNetConfig.tiny()
    unet = build_unet(cfg, seed=0, dtype=torch.float16, device="cuda")
    tools = (IdentityVAE(), unet, RandomTextEncoder(cfg.cross_attention_dim).cuda(), SimpleWordTokenizer(),
             LMSDiscreteScheduler(beta_start=0.00085, beta_end=0.012, beta_schedule="scaled_linear"))
    s = SETTINGS["cat_dog"]
    c = _colours()
    base = dict(color_context=dict(s["ctx"]), color_map_image=color_map_image("cat_dog", SIZE),
                input_prompt=s["prompt"], unconditional_input_prompt="blurry")
    two = {c[0]: "a small red lantern", c[-1]: "a tall green tree"}
    entries = [dict(base, seed=0),
               dict(base, seed=1, region_prompts=two),
               dict(base, seed=2, negative_region_prompts={c[0]: "dark", c[-1]: "dead leaves"}),
               dict(base, seed=3, region_prompts={c[0]: "a small red lantern"},
                    negative_region_prompts={c[-1]: "dead leaves"}, region_base_ratio=0.5)]
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


@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16], ids=["f16", "bf16"])
def test_negative_region_step_has_as_many_launches_as_a_plain_step_and_replays(dtype):
    pos, neg = _mixed()
    sch = _sch()
    cond, uncond = _encode("cuda", region_prompts=pos, negative=neg)
    _, s = _run_gpu([cond], [uncond], [_lat(0, sch)], WF_ZERO, sch, dtype=dtype)
    assert int(s._ctx["WMAP_INDEX"][0]) == -1 and s._ctx[C.REGION_ROWS_KEY].tolist() == [0, 1]
    graph, s = _run_gpu([cond], [uncond], [_lat(0, sch)], WF, _sch(), dtype=dtype)
    eager, _ = _run_gpu([cond], [uncond], [_lat(0, sch)], WF, _sch(), dtype=dtype, use_graph=False)
    pc, pu = _encode("cuda")
    _, plain = _run_gpu([pc], [pu], [_lat(0, sch)], WF, _sch(), dtype=dtype)
    assert s.native_launches_per_step is not None
    assert s.native_launches_per_step == plain.native_launches_per_step
    assert torch.isfinite(graph).all()
    assert (graph - eager).abs().max().item() <= 1e-3 * eager.abs().max().item()
