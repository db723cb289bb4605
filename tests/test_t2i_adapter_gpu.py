"""T2I-Adapter units on the GPU.

Kernel: `pww_adapter_residual_{f16,bf16}` is bitwise its torch statement `((a + b [+ bias]) + feat)` in the element type
at every SD1.5, SD2.1 and tiny encoder-level shape, for m = 1 and 8, feat_rows 0, m and 2m, with and without a bias, in
place and out of place; with no feature it is bitwise `pww_resnet_residual` (bias) and torch's add (no bias).  Loop:
`PwWSampler` with adapter units against `reference_adapter_loop` (rel RMSE < 3e-2, the bar of the ControlNet loop tests),
the bit-for-bit equalities of a never-active or weight-0 adapter and of attention recording, the one-time adapter
forward, the launch count of an adapter step, batching and the public API."""
import pytest
import torch
from PIL import Image

import paint_with_words_sd_b200 as P
from oracle import loop as oracle_loop
from oracle.adapter_loop import reference_adapter_loop
from paint_with_words_sd_b200 import _native, fused_ops
from paint_with_words_sd_b200.adapter import T2IAdapter, build_adapter, unet_level_sizes
from paint_with_words_sd_b200.controlnet import build_controlnet
from paint_with_words_sd_b200.pipeline import PwWSampler
from paint_with_words_sd_b200.unet import UNetConfig, build_unet
from tests.fixtures import SETTINGS, color_map_image
from tests.test_controlnet_gpu import (STEPS, TOL, WF, _encode, _extra, _hint, _latents, _pil_hint, _rel_rmse,
                                       _scheduler, _unpatch)

pytestmark = pytest.mark.gpu
DTYPES = [torch.float16, torch.bfloat16]
CL = torch.channels_last


# ---------------------------------------------------------------------------------------------------------------------
# the kernel
# ---------------------------------------------------------------------------------------------------------------------
def _levels(cfg, latent):
    return [(c, h, w) for c, (h, w) in zip(cfg.block_out_channels, unet_level_sizes(latent, latent))]


LEVELS = {"sd15": _levels(UNetConfig.sd15(), 64), "sd21": _levels(UNetConfig.sd21(), 96),
          "tiny": _levels(UNetConfig.tiny(), 16)}


def _t(rows, shape, dtype, g, scale=2.0):
    return (torch.randn(rows, *shape, generator=g, device="cuda") * scale).to(dtype).contiguous(memory_format=CL)


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("shape", sorted(LEVELS))
@pytest.mark.parametrize("m", [1, 8])
@pytest.mark.parametrize("feat_rows", ["0", "m", "2m"])
@pytest.mark.parametrize("bias", [False, True])
@pytest.mark.parametrize("in_place", [True, False])
def test_adapter_residual_is_bitwise_torch(dtype, shape, m, feat_rows, bias, in_place):
    B = 2 * m
    r = {"0": 0, "m": m, "2m": B}[feat_rows]
    g = torch.Generator(device="cuda").manual_seed(m * 10 + r)
    for level, s in enumerate(LEVELS[shape]):
        a, b = _t(B, s, dtype, g), _t(B, s, dtype, g)
        bv = torch.randn(s[0], generator=g, device="cuda") if bias else None
        feat = _t(r, s, dtype, g) if r else None
        ref = a + b if bv is None else (a.float() + b.float() + bv.view(1, -1, 1, 1)).to(dtype)
        if r:
            ref = torch.cat([ref[:r] + feat, ref[r:]], 0)
        out = None if in_place else torch.empty_like(b, memory_format=CL)
        n0 = _native.launch_count
        got = fused_ops.adapter_residual(a, b, bv, feat, out)
        torch.cuda.synchronize()
        assert _native.launch_count - n0 == 1
        assert got.data_ptr() == (b if in_place else out).data_ptr()
        assert torch.equal(got.view(torch.int16), ref.view(torch.int16)), \
            (level, (got.float() - ref.float()).abs().max().item())


@pytest.mark.parametrize("dtype", DTYPES)
def test_without_a_feature_it_is_the_resnet_epilogue_or_the_plain_add(dtype):
    g = torch.Generator(device="cuda").manual_seed(7)
    for s in LEVELS["sd15"]:
        a, b = _t(4, s, dtype, g), _t(4, s, dtype, g)
        bias = torch.randn(s[0], generator=g, device="cuda")
        want = fused_ops.resnet_residual(a, b, bias, out=torch.empty_like(b, memory_format=CL))
        got = fused_ops.adapter_residual(a, b, bias, None, torch.empty_like(b, memory_format=CL))
        assert torch.equal(got.view(torch.int16), want.view(torch.int16))
        got = fused_ops.adapter_residual(a, b, None, None, torch.empty_like(b, memory_format=CL))
        assert torch.equal(got.view(torch.int16), (a + b).view(torch.int16))


def test_mismatched_operands_raise_before_any_launch():
    g = torch.Generator(device="cuda").manual_seed(0)
    a, b = _t(2, (64, 4, 4), torch.float16, g), _t(2, (64, 4, 4), torch.float16, g)
    n0 = _native.launch_count
    bad = [
        dict(a=_t(2, (32, 4, 4), torch.float16, g)),
        dict(a=a.to(torch.bfloat16)),
        dict(a=a.contiguous()),
        dict(feat=_t(3, (64, 4, 4), torch.float16, g)),
        dict(feat=_t(1, (64, 2, 4), torch.float16, g)),
        dict(feat=_t(1, (64, 4, 4), torch.bfloat16, g)),
        dict(bias=torch.zeros(64, device="cuda", dtype=torch.float16)),
        dict(bias=torch.zeros(32, device="cuda")),
        dict(out=torch.empty(2, 64, 4, 4, device="cuda", dtype=torch.float16)),
    ]
    for kw in bad:
        args = {**dict(a=a, b=b, bias=None, feat=None, out=None), **kw}
        with pytest.raises(ValueError, match="adapter_residual"):
            fused_ops.adapter_residual(args["a"], args["b"], args["bias"], args["feat"], args["out"])
    assert _native.launch_count == n0


# ---------------------------------------------------------------------------------------------------------------------
# the loop
# ---------------------------------------------------------------------------------------------------------------------
def _units(spec, dtype, device):
    """spec: "full" / "light" / "net" per unit -> models of the tiny config, seeds by position."""
    cfg = UNetConfig.tiny()
    out = []
    for i, k in enumerate(spec):
        if k == "net":
            out.append(build_controlnet(cfg, seed=1 + i, dtype=dtype, device=device))
        else:
            out.append(build_adapter(cfg, k, 64 if k == "full" and i % 2 else 192, seed=3 + i, dtype=dtype,
                                     device=device))
    return out


def _reference(spec, weights, guesses=None, starts=None, ends=None, inpaint=False):
    cfg = UNetConfig.tiny(in_channels=9 if inpaint else 4)
    unet = build_unet(cfg, seed=0)
    units = _units(spec, torch.float32, "cpu")
    sch = _scheduler()
    cond, uncond = _encode(cfg, "aurora", "cpu")
    try:
        oracle_loop.patch_with_oracle(unet)
        return reference_adapter_loop(unet, units, [k != "net" for k in spec], sch, cond, uncond, _latents(0, sch), WF,
                                      [_hint(i) for i in range(len(spec))], 7.5, weights, guesses, starts, ends,
                                      extra_input=_extra() if inpaint else None)
    finally:
        _unpatch(unet)


def _gpu(units, dtype=torch.float16, use_graph=True, inpaint=False, record=False, **control):
    cfg = UNetConfig.tiny(in_channels=9 if inpaint else 4)
    unet = build_unet(cfg, seed=0, dtype=dtype, device="cuda")
    if units is not None:
        control.setdefault("control_image", [_hint(i) for i in range(len(units))] if isinstance(units, list)
                           else _hint(0))
    sch = _scheduler()
    cond, uncond = _encode(cfg, "aurora", "cuda")
    P.patch_unet(unet)
    try:
        s = PwWSampler(unet, sch, [cond], [uncond], _latents(0, sch).cuda(), WF, 7.5, use_graph=use_graph,
                       extra_input=_extra().cuda() if inpaint else None, controlnet=units, record_attention=record,
                       **control)
        out = s.run().float().cpu()
    finally:
        P.unpatch_all()
    return out, s


CASES = {
    "full": dict(spec=["full"], weights=[1.0]),
    "light": dict(spec=["light"], weights=[1.2]),
    "guess": dict(spec=["full"], weights=[0.9], guesses=[True]),
    "window": dict(spec=["full"], weights=[1.0], starts=[0.0], ends=[0.5]),
    "two_adapters": dict(spec=["full", "light"], weights=[0.8, 1.1]),
    "adapter_and_controlnet": dict(spec=["full", "net"], weights=[1.0, 0.7], starts=[0.0, 0.25], ends=[1.0, 1.0]),
    "inpaint": dict(spec=["full"], weights=[1.0], inpaint=True),
    "bf16": dict(spec=["full", "net"], weights=[1.0, 0.6], dtype=torch.bfloat16),
}


@pytest.mark.parametrize("case", sorted(CASES))
def test_sampler_matches_the_reference_loop(case):
    kw = dict(CASES[case])
    spec, dtype = kw.pop("spec"), kw.pop("dtype", torch.float16)
    ref = _reference(spec, **kw)
    n = len(spec)
    out, _ = _gpu(_units(spec, dtype, "cuda"), dtype, inpaint=kw.get("inpaint", False),
                  controlnet_conditioning_scale=kw["weights"], guess_mode=kw.get("guesses") or False,
                  control_guidance_start=kw.get("starts") or [0.0] * n, control_guidance_end=kw.get("ends") or [1.0] * n)
    assert torch.isfinite(out).all()
    err = _rel_rmse(out, ref)
    assert err < TOL, (case, err)


def test_an_adapter_changes_the_result():
    with_adapter, _ = _gpu(_units(["full"], torch.float16, "cuda"))
    without, _ = _gpu(None)
    light, _ = _gpu(_units(["light"], torch.float16, "cuda"))
    assert _rel_rmse(with_adapter, without) > TOL
    assert _rel_rmse(light, without) > TOL


@pytest.mark.parametrize("use_graph", [False, True])
def test_never_active_or_weight_zero_adapter_is_the_sampler_without_it_bit_for_bit(use_graph):
    plain, ps = _gpu(None, use_graph=use_graph)
    never, s = _gpu(_units(["full"], torch.float16, "cuda"), use_graph=use_graph, control_guidance_start=1.0)
    zero, _ = _gpu(_units(["full"], torch.float16, "cuda"), use_graph=use_graph, controlnet_conditioning_scale=0.0)
    assert torch.equal(never, plain) and torch.equal(zero, plain)
    assert s._adapter_sums == {}
    net_only, _ = _gpu(_units(["net"], torch.float16, "cuda"), use_graph=use_graph, controlnet_conditioning_scale=0.7)
    mixed, ms = _gpu(_units(["net", "full"], torch.float16, "cuda"), use_graph=use_graph,
                     controlnet_conditioning_scale=[0.7, 1.0], control_guidance_start=[0.0, 1.0])
    mixed0, _ = _gpu(_units(["net", "full"], torch.float16, "cuda"), use_graph=use_graph,
                     controlnet_conditioning_scale=[0.7, 0.0])
    assert torch.equal(mixed, net_only) and torch.equal(mixed0, net_only)


def test_record_attention_leaves_the_latents_unchanged():
    units = _units(["full", "net"], torch.float16, "cuda")
    off, _ = _gpu(units, controlnet_conditioning_scale=[1.0, 0.5])
    on, s = _gpu(units, record=True, controlnet_conditioning_scale=[1.0, 0.5])
    assert torch.equal(on, off)
    assert all(torch.isfinite(m).all() for m in s.attention_maps())


def test_the_adapter_runs_once_per_unit_and_never_inside_a_step():
    units = _units(["full", "light"], torch.float16, "cuda")
    calls = [0, 0]

    def hook(u):
        def f(*_):
            calls[u] += 1
        return f
    handles = [n.register_forward_hook(hook(u)) for u, n in enumerate(units)]
    try:
        _, s = _gpu(units, use_graph=False, control_guidance_start=[0.0, 0.5])
        assert s._step_no == STEPS and calls == [1, 1]
    finally:
        for h in handles:
            h.remove()


def test_an_adapter_only_step_has_the_plain_step_launches_plus_three():
    _, plain = _gpu(None)
    _, s = _gpu(_units(["full", "light"], torch.float16, "cuda"), control_guidance_start=[0.0, 0.5])
    launches = s.native_launches_per_active_set
    assert set(launches) == {(True, False), (True, True)}
    assert all(n == plain.native_launches_per_step + 3 for n in launches.values()), launches


def test_batched_images_with_their_own_hints_and_weights_match_solo_runs():
    cfg = UNetConfig.tiny()
    unet = build_unet(cfg, seed=0, dtype=torch.float16, device="cuda")
    units = _units(["full", "net"], torch.float16, "cuda")
    names = ["aurora", "cat_dog"]
    hints = [[_hint(0), _hint(1)], [_hint(2), _hint(3)]]         # [unit][image]
    weights = [[1.0, 0.6], [0.5, 1.3]]
    P.patch_unet(unet)
    try:
        sch = _scheduler()
        enc = [_encode(cfg, n, "cuda") for n in names]
        lat = torch.cat([_latents(i, sch) for i in range(2)], 0).cuda()
        batch = PwWSampler(unet, sch, [c for c, _ in enc], [u for _, u in enc], lat, WF, 7.5, controlnet=units,
                           control_image=hints, controlnet_conditioning_scale=weights,
                           control_guidance_end=[1.0, 0.5]).run().float().cpu()
        solo = []
        for i in range(2):
            sch = _scheduler()
            solo.append(PwWSampler(unet, sch, [enc[i][0]], [enc[i][1]], _latents(i, sch).cuda(), WF, 7.5,
                                   controlnet=units, control_image=[hints[0][i], hints[1][i]],
                                   controlnet_conditioning_scale=[weights[0][i], weights[1][i]],
                                   control_guidance_end=[1.0, 0.5]).run().float().cpu())
    finally:
        P.unpatch_all()
    for i in range(2):
        d = (batch[i] - solo[i][0]).abs().max().item()
        assert torch.isfinite(batch[i]).all() and d <= 2e-2 * solo[i].abs().max().item(), (i, d)


def test_public_api_with_adapters():
    tools = P.pww_load_tools("cuda:0", hf_model_path="synthetic:tiny")
    adapter = P.pww_load_adapter("synthetic:tiny:full192", device="cuda:0")
    assert isinstance(adapter, T2IAdapter)
    net = P.pww_load_controlnet("synthetic:tiny", device="cuda:0", seed=1)
    a, c = SETTINGS["aurora"], SETTINGS["cat_dog"]
    try:
        image = P.paint_with_words(color_context=dict(a["ctx"]), color_map_image=color_map_image("aurora", 128),
                                   input_prompt=a["prompt"], num_inference_steps=STEPS, device="cuda:0",
                                   preloaded_utils=tools, controlnet=adapter, control_image=_pil_hint(0, 128))
        entries = [dict(color_context=a["ctx"], color_map_image=color_map_image("aurora", 128),
                        input_prompt=a["prompt"], seed=0, control_image=[_pil_hint(0, 128), _pil_hint(1, 128)]),
                   dict(color_context=c["ctx"], color_map_image=color_map_image("cat_dog", 128),
                        input_prompt=c["prompt"], seed=1, control_image=[_pil_hint(2, 128), _pil_hint(3, 128)],
                        controlnet_conditioning_scale=[0.5, 1.2])]
        got = P.paint_with_words_batch(entries, num_inference_steps=3, device="cuda:0", preloaded_utils=tools,
                                       return_latents=True, controlnet=[adapter, net])
        pipe = P.PaintWithWord_StableDiffusionPipeline(*[tools[i] for i in (0, 2, 3, 1)], controlnet=[adapter, net])
        out = pipe(a["prompt"], color_map_image=color_map_image("aurora", 128), color_context=dict(a["ctx"]),
                   num_inference_steps=3, control_image=[_pil_hint(0, 128), _pil_hint(1, 128)], output_type="pil")
        itools = P.pww_load_tools("cuda:0", hf_model_path="synthetic:tiny-inpaint")
        inp = P.paint_with_words_inpaint(color_context=dict(a["ctx"]), color_map_image=color_map_image("aurora", 128),
                                         mask_image=Image.new("L", (128, 128), 255), init_image=_pil_hint(2, 128),
                                         input_prompt=a["prompt"], num_inference_steps=3, device="cuda:0",
                                         preloaded_utils=itools, controlnet=adapter, control_image=_pil_hint(0, 128),
                                         guess_mode=True)
    finally:
        P.unpatch_all()
    assert image.size == (128, 128) and inp.size == (128, 128)
    assert len(got) == 2 and all(torch.isfinite(x).all() for x in got)
    assert len(out.images) == 1 and out.images[0].size == (128, 128)
