"""Multi-ControlNet on the GPU.

Kernel: `pww_control_combine_{f16,bf16}` is bitwise the torch left fold `(r0 * s0).to(E) + (r1 * s1).to(E) + ...` at
the SD1.5, SD2.1 and tiny residual shapes, for U = 2, 3, 10 units, m = 1, 8, rows = B and B / 2, in place into unit 0's
residuals and out of place.  Loop: `PwWSampler(controlnet=[a, b])` with tiny ControlNets against
`reference_multi_controlnet_loop` (rel RMSE < 3e-2, the bar of the other loop tests), a weight-0 second unit and a
second unit that is never in its window against the single-ControlNet sampler bit for bit, launch accounting per
active set, guess-mode routing, batching and the public API."""
import pytest
import torch
from PIL import Image

import paint_with_words_sd_b200 as P
from oracle import loop as oracle_loop
from oracle.multi_controlnet_loop import reference_multi_controlnet_loop
from paint_with_words_sd_b200 import _native, fused_ops
from paint_with_words_sd_b200.controlnet import build_controlnet, residual_shapes
from paint_with_words_sd_b200.pipeline import PwWSampler
from paint_with_words_sd_b200.unet import UNetConfig, build_unet
from tests.fixtures import SETTINGS, color_map_image
from tests.test_controlnet_gpu import (SIZE, STEPS, TOL, WF, _Counting, _encode, _hint, _latents, _pil_hint, _rel_rmse,
                                       _scheduler, _unpatch)

pytestmark = pytest.mark.gpu
DTYPES = [torch.float16, torch.bfloat16]


# ---------------------------------------------------------------------------------------------------------------------
# the kernel
# ---------------------------------------------------------------------------------------------------------------------
SHAPES = {"sd15": residual_shapes(UNetConfig.sd15(), 64), "sd21": residual_shapes(UNetConfig.sd21(), 96),
          "tiny": residual_shapes(UNetConfig.tiny(), 16)}


def _cl(t):
    return t.contiguous(memory_format=torch.channels_last)


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("shape", sorted(SHAPES))
@pytest.mark.parametrize("units", [2, 3, 10])
@pytest.mark.parametrize("m", [1, 8])
@pytest.mark.parametrize("guess", [False, True])
@pytest.mark.parametrize("in_place", [True, False])
def test_combine_is_bitwise_the_torch_left_fold(dtype, shape, units, m, guess, in_place):
    rows = m if guess else 2 * m
    g = torch.Generator(device="cuda").manual_seed(units * 100 + m * 10 + guess)
    res = [[_cl((torch.randn(rows, *s, generator=g, device="cuda") * 3).to(dtype)) for s in SHAPES[shape]]
           for _ in range(units)]
    n = len(SHAPES[shape])
    scales = torch.rand(units, n, rows, generator=g, device="cuda") * 2 - 0.5
    ref = []
    for k in range(n):
        acc = None
        for u in range(units):
            p = (res[u][k] * scales[u, k].view(rows, 1, 1, 1)).to(dtype)     # r * s in fp32, rounded to dtype
            acc = p if acc is None else acc + p
        ref.append(acc)
    out = None if in_place else [torch.empty_like(r) for r in res[0]]
    keep = [r.clone() for r in res[1]]
    n0 = _native.launch_count
    got = fused_ops.control_combine(res, scales, out)
    torch.cuda.synchronize()
    assert _native.launch_count - n0 == 1
    if in_place:
        assert all(a.data_ptr() == b.data_ptr() for a, b in zip(got, res[0]))
    for k, (d, e) in enumerate(zip(got, ref)):
        assert torch.equal(d.view(torch.int16), e.view(torch.int16)), (k, (d.float() - e.float()).abs().max().item())
    for a, b in zip(res[1], keep):          # the other units' residuals are read only
        assert torch.equal(a.view(torch.int16), b.view(torch.int16))


def test_combine_rejects_mismatched_residuals():
    a = [_cl(torch.randn(2, 8, 4, 4, device="cuda").half())]
    with pytest.raises(ValueError, match="unit 1's residual 0"):
        fused_ops.control_combine([a, [_cl(torch.randn(2, 16, 4, 4, device="cuda").half())]],
                                  torch.ones(2, 1, 2, device="cuda"))
    with pytest.raises(ValueError, match="control scales"):
        fused_ops.control_combine([a, a], torch.ones(2, 1, 1, device="cuda"))


# ---------------------------------------------------------------------------------------------------------------------
# the loop
# ---------------------------------------------------------------------------------------------------------------------
def _reference(weights, guesses=(False, False), starts=(0.0, 0.0), ends=(1.0, 1.0)):
    cfg = UNetConfig.tiny()
    unet = build_unet(cfg, seed=0)
    nets = [build_controlnet(cfg, seed=1), build_controlnet(cfg, seed=2)]
    sch = _scheduler()
    cond, uncond = _encode(cfg, "aurora", "cpu")
    try:
        oracle_loop.patch_with_oracle(unet)
        return reference_multi_controlnet_loop(unet, nets, sch, cond, uncond, _latents(0, sch), WF,
                                               [_hint(0), _hint(1)], 7.5, weights, guesses, starts, ends)
    finally:
        _unpatch(unet)


def _gpu(nets=None, use_graph=True, **control):
    """The tiny UNet's sampler with `control` (PwWSampler's ControlNet keyword arguments); two ControlNets of seeds
    1 and 2 with hints 0 and 1 unless given."""
    cfg = UNetConfig.tiny()
    unet = build_unet(cfg, seed=0, dtype=torch.float16, device="cuda")
    if nets is None:
        nets = [build_controlnet(cfg, seed=s, dtype=torch.float16, device="cuda") for s in (1, 2)]
    control.setdefault("control_image", [_hint(0), _hint(1)][:len(nets)] if isinstance(nets, list) else _hint(0))
    sch = _scheduler()
    cond, uncond = _encode(cfg, "aurora", "cuda")
    P.patch_unet(unet)
    try:
        s = PwWSampler(unet, sch, [cond], [uncond], _latents(0, sch).cuda(), WF, 7.5, use_graph=use_graph,
                       controlnet=nets, **control)
        out = s.run().float().cpu()
    finally:
        P.unpatch_all()
    return out, s


CASES = {
    "full_windows": dict(weights=[1.0, 0.6]),
    "overlapping_windows": dict(weights=[0.8, 1.2], starts=[0.0, 0.25], ends=[0.5, 1.0]),
    "guess_mode_on_one_unit": dict(weights=[1.0, 0.8], guesses=[False, True]),
}


@pytest.mark.parametrize("case", sorted(CASES))
def test_sampler_matches_the_reference_loop(case):
    kw = CASES[case]
    ref = _reference(**kw)
    out, s = _gpu(controlnet_conditioning_scale=kw["weights"], guess_mode=kw.get("guesses", False),
                  control_guidance_start=kw.get("starts", 0.0), control_guidance_end=kw.get("ends", 1.0))
    assert torch.isfinite(out).all()
    err = _rel_rmse(out, ref)
    assert err < TOL, (case, err)
    single = _reference([kw["weights"][0], 0.0], kw.get("guesses", (False, False)))
    assert _rel_rmse(ref, single) > TOL          # the second unit matters at this bar


@pytest.mark.parametrize("use_graph", [False, True])
def test_a_weight_zero_second_unit_is_the_single_sampler_bit_for_bit(use_graph):
    cfg = UNetConfig.tiny()
    a = build_controlnet(cfg, seed=1, dtype=torch.float16, device="cuda")
    b = build_controlnet(cfg, seed=2, dtype=torch.float16, device="cuda")
    two, s = _gpu([a, b], use_graph, controlnet_conditioning_scale=[0.7, 0.0])
    one, _ = _gpu(a, use_graph, controlnet_conditioning_scale=0.7)
    assert torch.equal(two, one)
    if use_graph:
        assert set(s._graphs) == {(True, True)}


@pytest.mark.parametrize("use_graph", [False, True])
def test_a_second_unit_never_in_its_window_is_the_single_sampler_bit_for_bit(use_graph):
    """A step with one active unit of several runs no combine: the single ControlNet's step, bits and launches."""
    cfg = UNetConfig.tiny()
    a = build_controlnet(cfg, seed=1, dtype=torch.float16, device="cuda")
    b = build_controlnet(cfg, seed=2, dtype=torch.float16, device="cuda")
    two, s = _gpu([a, b], use_graph, controlnet_conditioning_scale=0.7, control_guidance_start=[0.0, 1.0],
                  control_guidance_end=[1.0, 1.0])
    one, single = _gpu(a, use_graph, controlnet_conditioning_scale=0.7)
    assert s._active_sets == [(True, False)] * STEPS
    assert torch.equal(two, one)
    if use_graph:
        assert s.native_launches_per_active_set == {(True, False): single.native_launches_per_step}
        assert s.native_launches_per_step is None


def _net_launches(net, s, unit):
    P.patch_unet(net)
    try:
        x = torch.randn(2, 4, SIZE // 8, SIZE // 8, device="cuda", dtype=torch.float16)
        before = _native.launch_count
        net(x, torch.tensor([500.0], device="cuda"), encoder_hidden_states=s._control_ctx,
            controlnet_cond_embedding=s._hints[unit])
        return _native.launch_count - before
    finally:
        P.unpatch_all()


def test_launch_accounting_per_active_set_and_its_size():
    """A step with active set A: the plain step + each active ControlNet's launches + the inject, and the combine
    before it when two or more units are active."""
    cfg = UNetConfig.tiny()
    nets = [build_controlnet(cfg, seed=s, dtype=torch.float16, device="cuda") for s in (1, 2)]
    _, s = _gpu(nets, control_guidance_start=[0.0, 0.25], control_guidance_end=[0.5, 0.75])
    plain = _plain_sampler()
    per_net = [_net_launches(net, s, u) for u, net in enumerate(nets)]
    assert all(n > 0 for n in per_net)
    assert s._active_sets == [(True, False), (True, True), (True, True), (False, True)]
    launches = s.native_launches_per_active_set
    assert set(launches) == {(True, False), (True, True), (False, True)} and len(s._graphs) == 3
    for a, got in launches.items():
        want = plain.native_launches_per_step + sum(n for n, on in zip(per_net, a) if on) + (2 if sum(a) > 1 else 1)
        assert got == want, (a, got, want)
    assert s.native_launches_per_step == launches[(True, True)]
    assert s.native_launches_per_step_without_control is None


def _plain_sampler():
    cfg = UNetConfig.tiny()
    unet = build_unet(cfg, seed=0, dtype=torch.float16, device="cuda")
    sch = _scheduler()
    cond, uncond = _encode(cfg, "aurora", "cuda")
    P.patch_unet(unet)
    try:
        s = PwWSampler(unet, sch, [cond], [uncond], _latents(0, sch).cuda(), WF, 7.5)
        s.run()
    finally:
        P.unpatch_all()
    return s


def test_guess_mode_on_one_unit_runs_every_controlnet_on_the_cond_rows():
    cfg = UNetConfig.tiny()
    nets = [build_controlnet(cfg, seed=s, dtype=torch.float16, device="cuda") for s in (1, 2)]
    counters = [_Counting(n) for n in nets]
    _gpu(nets, use_graph=False, guess_mode=[False, True])
    assert [c.batches for c in counters] == [[1] * STEPS, [1] * STEPS]
    counters = [_Counting(n) for n in nets]
    _gpu(nets, use_graph=False)
    assert [c.batches for c in counters] == [[2] * STEPS, [2] * STEPS]


def test_batched_images_with_per_unit_hints_and_weights_match_solo_runs():
    cfg = UNetConfig.tiny()
    unet = build_unet(cfg, seed=0, dtype=torch.float16, device="cuda")
    nets = [build_controlnet(cfg, seed=s, dtype=torch.float16, device="cuda") for s in (1, 2)]
    names = ["aurora", "cat_dog"]
    hints = [[_hint(0), _hint(1)], [_hint(2), _hint(3)]]         # [unit][image]
    weights = [[1.0, 0.6], [0.5, 1.3]]                            # [unit][image]
    P.patch_unet(unet)
    try:
        sch = _scheduler()
        enc = [_encode(cfg, n, "cuda") for n in names]
        lat = torch.cat([_latents(i, sch) for i in range(2)], 0).cuda()
        batch = PwWSampler(unet, sch, [c for c, _ in enc], [u for _, u in enc], lat, WF, 7.5, controlnet=nets,
                           control_image=hints, controlnet_conditioning_scale=weights,
                           control_guidance_end=[1.0, 0.5]).run().float().cpu()
        solo = []
        for i in range(2):
            sch = _scheduler()
            solo.append(PwWSampler(unet, sch, [enc[i][0]], [enc[i][1]], _latents(i, sch).cuda(), WF, 7.5,
                                   controlnet=nets, control_image=[hints[0][i], hints[1][i]],
                                   controlnet_conditioning_scale=[weights[0][i], weights[1][i]],
                                   control_guidance_end=[1.0, 0.5]).run().float().cpu())
    finally:
        P.unpatch_all()
    for i in range(2):
        d = (batch[i] - solo[i][0]).abs().max().item()
        assert torch.isfinite(batch[i]).all() and d <= 2e-2 * solo[i].abs().max().item(), (i, d)


def test_public_api_with_two_controlnets():
    tools = P.pww_load_tools("cuda:0", hf_model_path="synthetic:tiny")
    nets = [P.pww_load_controlnet("synthetic:tiny", device="cuda:0", seed=s) for s in (1, 2)]
    a, c = SETTINGS["aurora"], SETTINGS["cat_dog"]
    hints = [_pil_hint(0, 128), _pil_hint(1, 128)]
    entries = [
        dict(color_context=a["ctx"], color_map_image=color_map_image("aurora", 128), input_prompt=a["prompt"], seed=0,
             control_image=hints),
        dict(color_context=c["ctx"], color_map_image=color_map_image("cat_dog", 128), input_prompt=c["prompt"], seed=1,
             control_image=hints[::-1], controlnet_conditioning_scale=[0.5, 1.2]),
    ]
    try:
        got = P.paint_with_words_batch(entries, num_inference_steps=3, device="cuda:0", preloaded_utils=tools,
                                       return_latents=True, controlnet=nets, guess_mode=[False, True])
        refs = [P.paint_with_words(**dict(e, color_context=dict(e["color_context"])), num_inference_steps=3,
                                   device="cuda:0", preloaded_utils=tools, return_latents=True, controlnet=nets,
                                   guess_mode=[False, True])
                for e in entries]
        image = P.paint_with_words(**dict(entries[0], color_context=dict(a["ctx"])), num_inference_steps=2,
                                   device="cuda:0", preloaded_utils=tools, controlnet=nets,
                                   control_guidance_start=[0.0, 0.5], control_guidance_end=[0.5, 1.0])
        itools = P.pww_load_tools("cuda:0", hf_model_path="synthetic:tiny-inpaint")
        inp = P.paint_with_words_inpaint(color_context=dict(a["ctx"]), color_map_image=color_map_image("aurora", 128),
                                         mask_image=Image.new("L", (128, 128), 255), init_image=_pil_hint(2, 128),
                                         input_prompt=a["prompt"], num_inference_steps=3, device="cuda:0",
                                         preloaded_utils=itools, controlnet=nets, control_image=hints,
                                         controlnet_conditioning_scale=[1.0, 0.5])
        pipe = P.PaintWithWord_StableDiffusionPipeline(*[tools[i] for i in (0, 2, 3, 1)], controlnet=nets)
        out = pipe(a["prompt"], color_map_image=color_map_image("aurora", 128), color_context=dict(a["ctx"]),
                   num_inference_steps=3, control_image=hints, guess_mode=[False, True], output_type="pil")
        ipipe = P.PaintWithWord_StableDiffusionInpaintPipeline(*[itools[i] for i in (0, 2, 3, 1)], controlnet=nets)
        iout = ipipe(a["prompt"], image=_pil_hint(2, 128), mask_image=Image.new("L", (128, 128), 255),
                     color_map_image=color_map_image("aurora", 128), color_context=dict(a["ctx"]),
                     num_inference_steps=3, control_image=hints)
    finally:
        P.unpatch_all()
    for i, (x, ref) in enumerate(zip(got, refs)):
        d = (x.float() - ref.float()).abs().max().item()
        assert torch.isfinite(x).all() and d <= 2e-2 * ref.abs().max().item(), (i, d)
    assert image.size == (128, 128)
    assert inp.size == (128, 128)
    assert len(out.images) == 1 and out.images[0].size == (128, 128)
    assert len(iout.images) == 1 and iout.images[0].size == (128, 128)
