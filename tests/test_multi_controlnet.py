"""Multi-ControlNet on the CPU: the per-active-set scale tables, the active sets of overlapping, disjoint and closed
windows, argument validation of the sampler and every public entry point, `pww_control_combine_*` argument validation
(no GPU), the torch statement of the combine, and the oracle's consistency with the plain and single-ControlNet loops."""
import ctypes

import pytest
import torch
from PIL import Image

import paint_with_words_sd_b200 as P
from oracle import loop as oracle_loop
from oracle.controlnet_loop import reference_controlnet_loop
from oracle.multi_controlnet_loop import reference_multi_controlnet_loop
from paint_with_words_sd_b200 import _native
from paint_with_words_sd_b200 import pipeline as PL
from paint_with_words_sd_b200.controlnet import build_controlnet
from paint_with_words_sd_b200.scheduler import LMSDiscreteScheduler
from paint_with_words_sd_b200.unet import UNetConfig, attention_modules, build_unet, combine_control_residuals
from tests.fixtures import SETTINGS, color_map_image

CFG = UNetConfig.tiny()
WF = lambda w, sigma, qk: 0.4 * w * qk.max()     # noqa: E731
D = 0.825


@pytest.fixture(scope="module")
def models():
    """The tiny UNet and two ControlNets, fp32, with the oracle's attention."""
    unet, a, b = build_unet(CFG, seed=0), build_controlnet(CFG, seed=1), build_controlnet(CFG, seed=2)
    oracle_loop.patch_with_oracle(unet)
    yield unet, a, b
    cls = attention_modules(unet)[0].__class__
    if "__call__" in cls.__dict__:
        delattr(cls, "__call__")


def _sampler_inputs(m=1, size=64, steps=4):
    from paint_with_words_sd_b200.conditioning import _encode_text_color_inputs
    from paint_with_words_sd_b200.synthetic import RandomTextEncoder, SimpleWordTokenizer
    s = SETTINGS["aurora"]
    _, _, cond, uncond = _encode_text_color_inputs(RandomTextEncoder(CFG.cross_attention_dim), SimpleWordTokenizer(),
                                                   "cpu", color_map_image("aurora", size), dict(s["ctx"]), s["prompt"], "")
    sch = LMSDiscreteScheduler(beta_start=0.00085, beta_end=0.012, beta_schedule="scaled_linear")
    sch.set_timesteps(steps)
    lat = torch.randn(m, 4, size // 8, size // 8, generator=torch.manual_seed(0))
    return sch, [cond] * m, [uncond] * m, lat


def _imgs(k, size=64):
    return [torch.rand(1, 3, size, size, generator=torch.manual_seed(10 + i)) for i in range(k)]


def _f32(x):
    return torch.tensor(x, dtype=torch.float32).item()


def test_scale_tables_for_mixed_and_per_image_weights(models):
    unet, a, b = models
    sch, conds, unconds, lat = _sampler_inputs(m=2)
    s = PL.PwWSampler(unet, sch, conds, unconds, lat, WF, controlnet=[a, b], control_image=[_imgs(1)[0], _imgs(2)],
                      controlnet_conditioning_scale=[[0.5, 1.5], 0.25])
    assert "CONTROL_SCALES" not in s._ctx and not s.guess_mode
    assert list(s._combine_scales) == [(True, True)]
    t = s._combine_scales[(True, True)]
    assert tuple(t.shape) == (2, 13, 4) and t.dtype == torch.float32 and t.is_contiguous()
    # plain routing: rows [cond_0, cond_1, uncond_0, uncond_1], image i's weight in columns i and m + i
    assert torch.equal(t[0], torch.tensor([[0.5, 1.5, 0.5, 1.5]] * 13))
    assert torch.equal(t[1], torch.tensor([[0.25] * 4] * 13))
    assert len(s._hints) == 2 and tuple(s._hints[1].shape) == (4, 160, 8, 8)
    assert torch.equal(s._hints[0][:2], s._hints[0][2:])
    assert torch.equal(s._hints[1][:2], b.embed_condition(torch.cat(_imgs(2))))


def test_guess_mode_on_one_unit_routes_every_unit_to_the_cond_half(models):
    unet, a, b = models
    sch, conds, unconds, lat = _sampler_inputs(m=2)
    s = PL.PwWSampler(unet, sch, conds, unconds, lat, WF, controlnet=[a, b], control_image=[_imgs(1)[0]] * 2,
                      controlnet_conditioning_scale=[2.0, [0.5, 1.0]], guess_mode=[False, True])
    assert s.guess_mode
    t = s._combine_scales[(True, True)]
    assert tuple(t.shape) == (2, 13, 2)                     # rows = m: only the cond half gets residuals
    assert torch.equal(t[0], torch.full((13, 2), 2.0))      # unit 0 is not in guess mode: no decay
    for k in range(13):
        assert t[1, k].tolist() == [_f32(0.5 * D ** float(12 - k)), _f32(1.0 * D ** float(12 - k))]
    assert all(tuple(h.shape[:1]) == (2,) for h in s._hints)
    assert s._control_ctx["CONTEXT_TENSOR"].shape[0] == 2


@pytest.mark.parametrize("windows,sets", [
    # overlapping: [0, 0.5] and [0.25, 1] at 4 steps (i / n = 0, 0.25, 0.5, 0.75)
    (((0.0, 0.5), (0.25, 1.0)), [(True, False), (True, True), (True, True), (False, True)]),
    # disjoint
    (((0.0, 0.25), (0.5, 1.0)), [(True, False), (True, False), (False, True), (False, True)]),
    # one closed, one partly
    (((0.9, 0.95), (0.5, 0.5)), [(False, False), (False, False), (False, True), (False, False)]),
    # both closed
    (((0.9, 0.95), (0.8, 0.85)), [(False, False)] * 4),
])
def test_active_sets_and_their_tables(models, windows, sets):
    unet, a, b = models
    sch, conds, unconds, lat = _sampler_inputs()
    s = PL.PwWSampler(unet, sch, conds, unconds, lat, WF, controlnet=[a, b], control_image=_imgs(2),
                      controlnet_conditioning_scale=[0.5, 2.0], control_guidance_start=[w[0] for w in windows],
                      control_guidance_end=[w[1] for w in windows])
    assert s._active_sets == sets
    assert s._control_active == [any(x) for x in sets]
    assert set(s._combine_scales) == {x for x in sets if any(x)}
    for x, t in s._combine_scales.items():
        want = [w for w, on in zip([0.5, 2.0], x) if on]
        assert tuple(t.shape) == (len(want), 13, 2) and t.is_contiguous()
        assert torch.equal(t, torch.tensor(want)[:, None, None].expand(len(want), 13, 2))


def test_a_list_of_one_sets_up_as_one_controlnet(models):
    unet, a, _ = models
    sch, conds, unconds, lat = _sampler_inputs(m=2)
    img = _imgs(1)[0]
    one = PL.PwWSampler(unet, sch, conds, unconds, lat, WF, controlnet=[a], control_image=[img],
                        controlnet_conditioning_scale=[0.7], guess_mode=[True], control_guidance_start=[0.25])
    single = PL.PwWSampler(unet, sch, conds, unconds, lat, WF, controlnet=a, control_image=img,
                           controlnet_conditioning_scale=0.7, guess_mode=True, control_guidance_start=0.25)
    assert one.controlnet == [a] and single.controlnet is a and one._nets == single._nets == [a]
    assert list(one._combine_scales) == list(single._combine_scales) == [(True,)]
    assert torch.equal(one._combine_scales[(True,)], single._combine_scales[(True,)])
    assert torch.equal(one._combine_scales[(True,)], PL.control_scales([0.7, 0.7], True)[None])
    assert one._active_sets == single._active_sets == [(False,), (True,), (True,), (True,)]
    assert len(one._hints) == len(single._hints) == 1 and torch.equal(one._hints[0], single._hints[0])


def test_sampler_rejects_bad_multi_control_arguments(models):
    unet, a, b = models
    sch, conds, unconds, lat = _sampler_inputs(m=2)
    imgs = _imgs(2)

    def make(**kw):
        args = dict(controlnet=[a, b], control_image=imgs)
        args.update(kw)
        return PL.PwWSampler(unet, sch, conds, unconds, lat, WF, **args)
    with pytest.raises(ValueError, match="controlnet: a list of 1 to 10"):
        make(controlnet=[a] * 11, control_image=[imgs[0]] * 11)
    with pytest.raises(ValueError, match="controlnet: a list of 1 to 10"):
        make(controlnet=[], control_image=[])
    with pytest.raises(ValueError, match="control_image must be a list of 2"):
        make(control_image=imgs[:1])
    with pytest.raises(ValueError, match="control_image must be a list of 2"):
        make(control_image=imgs[0])
    with pytest.raises(ValueError, match="control_image must be a list of 2"):
        make(control_image=None)
    with pytest.raises(ValueError, match=r"control_image\[1\]"):
        make(control_image=[imgs[0], [imgs[1]] * 3])
    with pytest.raises(ValueError, match=r"control_image\[0\] 0 is"):
        make(control_image=[torch.rand(1, 3, 32, 32), imgs[1]])
    with pytest.raises(ValueError, match="controlnet_conditioning_scale must be one value or a list of 2"):
        make(controlnet_conditioning_scale=[1.0, 0.5, 0.2])
    with pytest.raises(ValueError, match=r"controlnet_conditioning_scale\[1\]"):
        make(controlnet_conditioning_scale=[1.0, [0.5, 0.2, 0.1]])
    with pytest.raises(ValueError, match="guess_mode must be one value or a list of 2"):
        make(guess_mode=[True])
    with pytest.raises(ValueError, match="control_guidance_start must be one value or a list of 2"):
        make(control_guidance_start=[0.0, 0.1, 0.2])
    with pytest.raises(ValueError, match="control_guidance_end must be one value or a list of 2"):
        make(control_guidance_end=[1.0])
    with pytest.raises(ValueError, match=r"control_guidance_start\[1\] \(0.8\) must not exceed"):
        make(control_guidance_start=[0.0, 0.8], control_guidance_end=[1.0, 0.2])
    with pytest.raises(ValueError, match=r"controlnet\[1\] config cross_attention_dim"):
        make(controlnet=[a, build_controlnet(UNetConfig(block_out_channels=CFG.block_out_channels,
                                                        cross_attention_dim=32, attention_heads=4,
                                                        norm_num_groups=8))])
    with pytest.raises(ValueError, match=r"controlnet\[0\] config in_channels"):
        make(controlnet=[build_controlnet(UNetConfig.tiny(in_channels=9)), b])
    with pytest.raises(TypeError, match=r"controlnet\[1\] must be"):
        make(controlnet=[a, unet])


def test_the_same_model_twice_shares_its_kv_cache(models):
    unet, a, _ = models
    sch, conds, unconds, lat = _sampler_inputs()
    s = PL.PwWSampler(unet, sch, conds, unconds, lat, WF, controlnet=[a, a], control_image=_imgs(2))
    assert s._nets == [a, a] and len(s._hints) == 2 and not torch.equal(s._hints[0], s._hints[1])
    assert isinstance(s._control_ctx["KV_CACHE"], dict)


def test_public_api_rejects_bad_multi_control_arguments(models):
    unet, a, b = models
    cmap = color_map_image("aurora", 64)
    hint = Image.new("RGB", (64, 64))
    with pytest.raises(ValueError, match="control_image must be a list of 2"):
        P.paint_with_words(color_map_image=cmap, controlnet=[a, b], control_image=hint, preloaded_utils=())
    with pytest.raises(ValueError, match=r"control_image\[1\] is \(32, 64\)"):
        P.paint_with_words(color_map_image=cmap, controlnet=[a, b], control_image=[hint, Image.new("RGB", (32, 64))],
                           preloaded_utils=())
    with pytest.raises(ValueError, match=r"control_image\[0\]"):
        P.paint_with_words(color_map_image=cmap, controlnet=[a, b], control_image=[None, hint], preloaded_utils=())
    with pytest.raises(ValueError, match="controlnet_conditioning_scale"):
        P.paint_with_words(color_map_image=cmap, controlnet=[a, b], control_image=[hint, hint],
                           controlnet_conditioning_scale=[1.0, 1.0, 1.0], preloaded_utils=())
    with pytest.raises(ValueError, match="guess_mode"):
        P.paint_with_words(color_map_image=cmap, controlnet=[a, b], control_image=[hint, hint], guess_mode=[True],
                           preloaded_utils=())
    with pytest.raises(ValueError, match="controlnet: a list of 1 to 10"):
        P.paint_with_words(color_map_image=cmap, controlnet=[a] * 11, control_image=[hint] * 11, preloaded_utils=())
    with pytest.raises(ValueError, match=r"control_image\[1\]"):
        P.paint_with_words_inpaint(color_map_image=cmap, init_image=Image.new("RGB", (64, 64)), controlnet=[a, b],
                                   control_image=[hint, Image.new("RGB", (128, 128))], preloaded_utils=())
    with pytest.raises(ValueError, match="control_guidance_end"):
        P.paint_with_words_inpaint(color_map_image=cmap, init_image=Image.new("RGB", (64, 64)), controlnet=[a, b],
                                   control_image=[hint, hint], control_guidance_end=[1.0] * 3, preloaded_utils=())
    base = dict(color_context=dict(SETTINGS["aurora"]["ctx"]), color_map_image=cmap)
    with pytest.raises(ValueError, match=r"settings\[1\].*control_image must be a list of 2"):
        P.paint_with_words_batch([dict(base, control_image=[hint, hint]), dict(base, control_image=[hint])],
                                 controlnet=[a, b], preloaded_utils=())
    with pytest.raises(ValueError, match=r"settings\[0\].*controlnet_conditioning_scale"):
        P.paint_with_words_batch([dict(base, control_image=[hint, hint], controlnet_conditioning_scale=[1.0])],
                                 controlnet=[a, b], preloaded_utils=())
    with pytest.raises(ValueError, match=r"settings\[0\].*control_guidance_start"):
        P.paint_with_words_batch([dict(base, control_image=[hint, hint])], controlnet=[a, b],
                                 control_guidance_start=[0.0, 0.1, 0.2], preloaded_utils=())
    for cls in (P.PaintWithWord_StableDiffusionPipeline, P.PaintWithWord_StableDiffusionInpaintPipeline):
        pipe = cls.__new__(cls)
        pipe.controlnet = [a, b]
        assert pipe._control([hint, hint], [0.5, 1.0], [False, True], 0.0, [1.0, 0.5]) == dict(
            controlnet=[a, b], control_image=[hint, hint], controlnet_conditioning_scale=[0.5, 1.0],
            guess_mode=[False, True], control_guidance_start=0.0, control_guidance_end=[1.0, 0.5])


def test_combine_statement_is_the_left_fold_in_the_element_type():
    g = torch.Generator().manual_seed(0)
    shapes = [(8, 4, 4), (16, 2, 2)]
    for dtype in (torch.float32, torch.float16, torch.bfloat16):
        units = [[(torch.randn(2, *s, generator=g) * 3).to(dtype) for s in shapes] for _ in range(3)]
        scales = torch.rand(3, 2, 2, generator=g) * 2
        got = combine_control_residuals(units, scales)
        for k in range(2):
            want = None
            for u in range(3):
                p = (units[u][k].float() * scales[u, k].view(2, 1, 1, 1)).to(dtype)
                want = p if want is None else (want.float() + p.float()).to(dtype)
            assert got[k].dtype == dtype and torch.equal(got[k], want), (dtype, k)


# ---------------------------------------------------------------------------------------------------------------------
# the oracle's own consistency
# ---------------------------------------------------------------------------------------------------------------------
def _oracle_runs(unet, fn):
    try:
        oracle_loop.patch_with_oracle(unet)
        return fn()
    finally:
        cls = attention_modules(unet)[0].__class__
        if "__call__" in cls.__dict__:
            delattr(cls, "__call__")


def test_oracle_with_every_window_closed_is_the_plain_loop(models):
    unet, a, b = models
    sch, conds, unconds, lat = _sampler_inputs()
    plain, closed = _oracle_runs(unet, lambda: (
        oracle_loop.reference_denoise_loop(unet, sch, dict(conds[0]), dict(unconds[0]), lat, WF, 7.5),
        reference_multi_controlnet_loop(unet, [a, b], sch, dict(conds[0]), dict(unconds[0]), lat, WF, _imgs(2),
                                        control_guidance_starts=[0.9, 0.8], control_guidance_ends=[0.95, 0.85])))
    assert torch.equal(plain, closed)


@pytest.mark.parametrize("guess", [False, True])
def test_oracle_with_one_unit_is_the_single_controlnet_loop(models, guess):
    unet, a, _ = models
    sch, conds, unconds, lat = _sampler_inputs()
    img = _imgs(1)[0]
    single, multi = _oracle_runs(unet, lambda: (
        reference_controlnet_loop(unet, a, sch, dict(conds[0]), dict(unconds[0]), lat, WF, img, 7.5, 0.7, guess,
                                  0.25, 1.0),
        reference_multi_controlnet_loop(unet, [a], sch, dict(conds[0]), dict(unconds[0]), lat, WF, [img], 7.5, [0.7],
                                        [guess], [0.25], [1.0])))
    assert torch.equal(single, multi)


def test_oracle_second_unit_changes_the_result(models):
    unet, a, b = models
    sch, conds, unconds, lat = _sampler_inputs()
    img = _imgs(2)
    one, two = _oracle_runs(unet, lambda: (
        reference_multi_controlnet_loop(unet, [a], sch, dict(conds[0]), dict(unconds[0]), lat, WF, img[:1]),
        reference_multi_controlnet_loop(unet, [a, b], sch, dict(conds[0]), dict(unconds[0]), lat, WF, img)))
    assert not torch.allclose(one, two, rtol=3e-2, atol=1e-3)


# ---------------------------------------------------------------------------------------------------------------------
# pww_control_combine_{f16,bf16}: validation before any CUDA call
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name", ["pww_control_combine_f16", "pww_control_combine_bf16"])
def test_control_combine_rejects_bad_arguments_without_gpu(name):
    fn = getattr(_native.lib(), name)
    buf = (ctypes.c_char * 4096)()
    p16 = (ctypes.addressof(buf) + 15) // 16 * 16

    def call(units=2, n=2, out=None, res=None, elems=None, rows=1, scales=p16 + 1024, count=None):
        k = n if count is None else count
        u = units if count is None else 1
        o = (ctypes.c_void_p * max(k, 1))(*([p16] * k if out is None else out))
        r = (ctypes.c_void_p * max(u * k, 1))(*([p16 + 512] * (u * k) if res is None else res))
        e = (ctypes.c_int64 * max(k, 1))(*([16] * k if elems is None else elems))
        return fn(units, n, o, r, e, rows, scales, None)
    assert call(units=0, count=1) == -1
    assert call(units=11, count=1) == -1
    assert call(units=-1, count=1) == -1
    assert call(n=0, count=1) == -1
    assert call(n=17, count=1) == -1
    assert call(rows=0) == -1
    assert call(rows=-3) == -1
    assert call(scales=None) == -1
    assert call(elems=[16, 0]) == -1
    assert call(elems=[-8, 16]) == -1
    assert call(elems=[16, 12]) == -1
    assert call(out=[p16, None]) == -1
    assert call(out=[p16, p16 + 8]) == -1
    assert call(res=[p16, p16, p16, None]) == -1
    assert call(res=[p16, p16 + 2, p16, p16]) == -1
    assert fn(2, 1, None, None, None, 1, p16, None) == -1
