"""ControlNet on the CPU: the model's residual shapes and hint path, the UNet's residual path against a restatement of
the extension's injection (pww_controlnet/scripts/hook_pww.py:166-175), the CONTROL_SCALES table, the guidance window,
argument validation of the sampler and the public API, and `pww_control_inject_*` argument validation (no GPU)."""
import ctypes
import inspect

import pytest
import torch
from PIL import Image

import paint_with_words_sd_b200 as P
from oracle import loop as oracle_loop
from oracle.controlnet_loop import reference_controlnet_loop
from paint_with_words_sd_b200 import _native
from paint_with_words_sd_b200 import pipeline as PL
from paint_with_words_sd_b200.controlnet import ControlNetModel, build_controlnet, pww_load_controlnet
from paint_with_words_sd_b200.scheduler import LMSDiscreteScheduler
from paint_with_words_sd_b200.unet import UNetConfig, attention_modules, build_unet, timestep_embedding
from tests.fixtures import SETTINGS, color_map_image

CFG = UNetConfig.tiny()
T_STEP = 500.0


@pytest.fixture(scope="module")
def models():
    """The tiny UNet and ControlNet, fp32, with the oracle's attention (which takes tensor and dict contexts)."""
    unet, net = build_unet(CFG, seed=0), build_controlnet(CFG, seed=1)
    oracle_loop.patch_with_oracle(unet)
    yield unet, net
    cls = attention_modules(unet)[0].__class__
    if "__call__" in cls.__dict__:
        delattr(cls, "__call__")


def _plain(ctx, **extra):
    """An unbiased PwW context dict around a text context tensor."""
    d = {"CONTEXT_TENSOR": ctx, "CROSS_ATTENTION_WEIGHT_ORIG": 0, "WEIGHT_FUNCTION": lambda w, sigma, qk: 0.0,
         "SIGMA": 1.0}
    d.update(extra)
    return d


def _inputs(b=1, size=16, seed=0):
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(b, 4, size, size, generator=g)
    ctx = torch.randn(b, 77, CFG.cross_attention_dim, generator=g)
    hint = torch.rand(b, 3, 8 * size, 8 * size, generator=g)
    return x, ctx, hint


def _unet_skips(unet, x, ctx):
    """The UNet's 12 skips and its mid-block output, read with forward hooks."""
    got = []
    hooks = [unet.conv_in.register_forward_hook(lambda m, i, o: got.append(o))]
    hooks += [b.register_forward_hook(lambda m, i, o: got.extend(o[1])) for b in unet.down_blocks]
    hooks.append(unet.mid_block.register_forward_hook(lambda m, i, o: got.append(o)))
    try:
        unet(x, T_STEP, encoder_hidden_states=ctx)
    finally:
        for h in hooks:
            h.remove()
    return got


def test_residual_shapes_equal_the_unet_skips_and_mid_output(models):
    unet, net = models
    x, ctx, hint = _inputs()
    down, mid = net(x, T_STEP, ctx, controlnet_cond=hint, return_dict=False)
    skips = _unet_skips(unet, x, ctx)
    assert len(down) == 12 and len(skips) == 13
    assert [tuple(r.shape) for r in down] + [tuple(mid.shape)] == [tuple(s.shape) for s in skips]


def test_parameter_names_follow_diffusers(models):
    names = {n.split(".")[0] for n, _ in models[1].named_parameters()}
    assert names == {"conv_in", "time_embedding", "controlnet_cond_embedding", "down_blocks", "mid_block",
                     "controlnet_down_blocks", "controlnet_mid_block"}
    emb = {n for n, _ in models[1].controlnet_cond_embedding.named_parameters()}
    assert emb == {f"{p}.{w}" for p in ["conv_in", "conv_out"] + [f"blocks.{i}" for i in range(6)]
                   for w in ("weight", "bias")}
    assert len(models[1].controlnet_down_blocks) == 12
    # the hint block: 3 -> 16 -> 16 -> 32 -> 32 -> 96 -> 96 -> 256 -> C0, three stride-2 convs
    convs = [models[1].controlnet_cond_embedding.conv_in, *models[1].controlnet_cond_embedding.blocks,
             models[1].controlnet_cond_embedding.conv_out]
    assert [c.in_channels for c in convs] + [convs[-1].out_channels] == [3, 16, 16, 32, 32, 96, 96, 256, 160]
    assert [c.stride[0] for c in convs] == [1, 1, 2, 1, 2, 1, 2, 1]


def test_zero_convs_and_hint_output_have_random_weights(models):
    net = models[1]
    for conv in list(net.controlnet_down_blocks) + [net.controlnet_mid_block, net.controlnet_cond_embedding.conv_out]:
        assert conv.weight.abs().sum() > 0


def test_hint_image_and_its_embedding_give_the_same_bits(models):
    _, net = models
    x, ctx, hint = _inputs(b=2, seed=3)
    a = net(x, T_STEP, ctx, controlnet_cond=hint)
    b = net(x, T_STEP, ctx, controlnet_cond_embedding=net.embed_condition(hint))
    for ra, rb in zip(list(a.down_block_res_samples) + [a.mid_block_res_sample],
                      list(b.down_block_res_samples) + [b.mid_block_res_sample]):
        assert torch.equal(ra, rb)
    with pytest.raises(ValueError, match="exactly one"):
        net(x, T_STEP, ctx)
    with pytest.raises(ValueError, match="exactly one"):
        net(x, T_STEP, ctx, controlnet_cond=hint, controlnet_cond_embedding=net.embed_condition(hint))


def _restated_forward(unet, x, ctx, control, control_scales):
    """hook_pww.py:151-179 over this UNet's blocks: the encoder, `h = mid + control.pop()` scaled, then every decoder
    stage takes `cat([h, hs.pop() + control.pop()])`.  Rows beyond the residuals' batch get nothing (cfg_based_adder in
    guess mode)."""
    temb = timestep_embedding(torch.tensor([T_STEP]).expand(x.shape[0]), CFG.block_out_channels[0])
    temb = unet.time_embedding["linear_2"](torch.nn.functional.silu(unet.time_embedding["linear_1"](temb)))
    h = unet.conv_in(x)
    hs = [h]
    for blk in unet.down_blocks:
        h, outs = blk(h, temb, ctx)
        hs.extend(outs)
    h = unet.mid_block(h, temb, ctx)
    control = [c * s.view(-1, 1, 1, 1) for c, s in zip(control, control_scales)]

    def adder(base, c):
        rows = c.shape[0]
        return torch.cat([base[:rows] + c, base[rows:]], 0)
    h = adder(h, control.pop())
    hs = [adder(s, c) for s, c in zip(hs, control)]
    for blk in unet.up_blocks:
        h = blk(h, hs, temb, ctx)
    return unet.conv_out(torch.nn.functional.silu(unet.conv_norm_out(h)))


@pytest.mark.parametrize("guess", [False, True])
def test_unet_residual_path_equals_the_restated_injection(models, guess):
    unet, net = models
    x, ctx, hint = _inputs(b=2, seed=5)
    rows = 1 if guess else 2
    down, mid = net(x[:rows], T_STEP, ctx[:rows], controlnet_cond=hint[:rows], return_dict=False)
    scales = PL.control_scales([0.7], guess)          # [13, 2] plain (m = 1: cond and uncond), [13, 1] guess mode
    assert tuple(scales.shape) == (13, rows)
    with torch.no_grad():
        got = unet(x, T_STEP, encoder_hidden_states=_plain(ctx, CONTROL_SCALES=scales),
                   down_block_additional_residuals=down, mid_block_additional_residual=mid).sample
        ref = _restated_forward(unet, x, _plain(ctx), list(down) + [mid], list(scales))
        plain = unet(x, T_STEP, encoder_hidden_states=_plain(ctx)).sample
    assert torch.allclose(got, ref, rtol=1e-5, atol=1e-5)      # fp32: the same ops, the last bits may differ
    assert not torch.allclose(got[:rows], plain[:rows], rtol=1e-2, atol=1e-3)
    if guess:
        assert torch.equal(got[1:], plain[1:])           # the uncond half gets nothing


def test_zero_residuals_change_no_bit(models):
    unet, net = models
    x, ctx, _ = _inputs(b=2, seed=6)
    skips = _unet_skips(unet, x, ctx)
    zeros = [torch.zeros_like(s) for s in skips]
    with torch.no_grad():
        plain = unet(x, T_STEP, encoder_hidden_states=ctx).sample
        got = unet(x, T_STEP, encoder_hidden_states=ctx, down_block_additional_residuals=zeros[:-1],
                   mid_block_additional_residual=zeros[-1]).sample
        with pytest.raises(ValueError, match="go together"):
            unet(x, T_STEP, encoder_hidden_states=ctx, down_block_additional_residuals=zeros[:-1])
    assert torch.equal(got, plain)


def test_control_scales_table():
    plain = PL.control_scales([0.5, 2.0], guess_mode=False)
    assert plain.dtype == torch.float32 and tuple(plain.shape) == (13, 4)
    assert torch.equal(plain, torch.tensor([[0.5, 2.0, 0.5, 2.0]] * 13))
    guess = PL.control_scales([0.5, 2.0], guess_mode=True)
    assert tuple(guess.shape) == (13, 2)
    for k in range(13):
        for i, w in enumerate([0.5, 2.0]):
            assert guess[k, i].item() == torch.tensor(w * 0.825 ** float(12 - k), dtype=torch.float32).item()
    assert guess[12].tolist() == [0.5, 2.0]


@pytest.mark.parametrize("start,end", [(0.0, 1.0), (0.25, 0.75), (0.0, 0.5), (0.5, 1.0), (0.1, 0.1), (0.3, 0.31),
                                       (0.05, 0.95), (1.0, 1.0)])
def test_guidance_window_rule_at_20_steps(start, end):
    n = 20
    got = [PL.control_step_active(i, n, start, end) for i in range(n)]
    assert got == [start <= i / n <= end for i in range(n)]
    # boundaries: i/n exactly at start or end is inside
    for i in range(n):
        if i / n in (start, end):
            assert got[i]
    if (start, end) == (0.25, 0.75):
        assert [i for i in range(n) if got[i]] == list(range(5, 16))
    if (start, end) == (1.0, 1.0):
        assert not any(got)


def _sampler_inputs(m=1, size=64):
    from paint_with_words_sd_b200.conditioning import _encode_text_color_inputs
    from paint_with_words_sd_b200.synthetic import RandomTextEncoder, SimpleWordTokenizer
    s = SETTINGS["aurora"]
    _, _, cond, uncond = _encode_text_color_inputs(RandomTextEncoder(CFG.cross_attention_dim), SimpleWordTokenizer(),
                                                   "cpu", color_map_image("aurora", size), dict(s["ctx"]), s["prompt"], "")
    sch = LMSDiscreteScheduler(beta_start=0.00085, beta_end=0.012, beta_schedule="scaled_linear")
    sch.set_timesteps(4)
    lat = torch.randn(m, 4, size // 8, size // 8, generator=torch.manual_seed(0))
    return sch, [cond] * m, [uncond] * m, lat


WF = lambda w, sigma, qk: 0.4 * w * qk.max()     # noqa: E731


def test_sampler_builds_one_controlnets_state_on_the_cpu(models):
    unet, net = models
    sch, conds, unconds, lat = _sampler_inputs(m=2)
    imgs = [torch.rand(1, 3, 64, 64, generator=torch.manual_seed(i)) for i in range(2)]
    s = PL.PwWSampler(unet, sch, conds, unconds, lat, WF, controlnet=net, control_image=imgs,
                      controlnet_conditioning_scale=[0.5, 1.5], control_guidance_start=0.25,
                      control_guidance_end=0.5)
    assert s._control_active == [False, True, True, False]
    # one active unit: its table is the inject's CONTROL_SCALES, which the step puts into the context
    assert list(s._combine_scales) == [(True,)] and "CONTROL_SCALES" not in s._ctx
    assert torch.equal(s._combine_scales[(True,)], PL.control_scales([0.5, 1.5], False)[None])
    hint = s._hints[0]
    assert len(s._hints) == 1 and tuple(hint.shape) == (4, 160, 8, 8)
    assert torch.equal(hint[:2], hint[2:]) and torch.equal(hint[:2], net.embed_condition(torch.cat(imgs)))
    assert s._control_ctx["CONTEXT_TENSOR"].data_ptr() == s._ctx["CONTEXT_TENSOR"].data_ptr()
    g = PL.PwWSampler(unet, sch, conds, unconds, lat, WF, controlnet=net, control_image=imgs[0], guess_mode=True)
    assert tuple(g._hints[0].shape) == (2, 160, 8, 8) and g._control_ctx["CONTEXT_TENSOR"].shape[0] == 2
    assert torch.equal(g._combine_scales[(True,)], PL.control_scales([1.0, 1.0], True)[None])


class _NoResidualUNet(torch.nn.Module):
    def __init__(self, unet):
        super().__init__()
        self.inner, self.config, self.in_channels = unet, unet.config, unet.in_channels

    def forward(self, sample, timestep, encoder_hidden_states=None):
        return self.inner(sample, timestep, encoder_hidden_states)


def test_sampler_rejects_bad_control_arguments(models):
    unet, net = models
    sch, conds, unconds, lat = _sampler_inputs(m=2)
    img = torch.rand(1, 3, 64, 64)

    def make(**kw):
        args = dict(controlnet=net, control_image=img)
        args.update(kw)
        return PL.PwWSampler(args.pop("unet", unet), sch, conds, unconds, lat, WF, **args)
    with pytest.raises(TypeError, match="controlnet"):
        make(controlnet=unet)
    with pytest.raises(TypeError, match="down_block_additional_residuals"):
        make(unet=_NoResidualUNet(unet))
    with pytest.raises(ValueError, match="cross_attention_dim"):
        make(controlnet=build_controlnet(UNetConfig(block_out_channels=CFG.block_out_channels, cross_attention_dim=32,
                                                    attention_heads=4, norm_num_groups=8)))
    with pytest.raises(ValueError, match="block_out_channels"):
        make(controlnet=build_controlnet(UNetConfig(block_out_channels=(80, 160, 320, 320), cross_attention_dim=64,
                                                    attention_heads=4, norm_num_groups=8)))
    with pytest.raises(ValueError, match="in_channels"):
        make(controlnet=build_controlnet(UNetConfig.tiny(in_channels=9)))
    with pytest.raises(ValueError, match="control_image"):
        make(control_image=torch.rand(1, 3, 32, 32))
    with pytest.raises(ValueError, match="control_image"):
        make(control_image=[img, img, img])
    with pytest.raises(ValueError, match="control_image"):
        make(control_image=None)
    with pytest.raises(ValueError, match="controlnet_conditioning_scale"):
        make(controlnet_conditioning_scale=[1.0, 0.5, 0.2])
    with pytest.raises(ValueError, match="control_guidance_start"):
        make(control_guidance_start=0.8, control_guidance_end=0.2)
    with pytest.raises(ValueError, match="controlnet is None"):
        make(controlnet=None)


def test_public_api_rejects_bad_control_images(models):
    unet, net = models
    cmap = color_map_image("aurora", 64)
    with pytest.raises(ValueError, match="control_image"):
        P.paint_with_words(color_map_image=cmap, controlnet=net, control_image=Image.new("RGB", (32, 64)),
                           preloaded_utils=())
    with pytest.raises(ValueError, match="control_image"):
        P.paint_with_words(color_map_image=cmap, controlnet=net, preloaded_utils=())
    with pytest.raises(ValueError, match="control_image"):
        P.paint_with_words_inpaint(color_map_image=cmap, init_image=Image.new("RGB", (64, 64)), controlnet=net,
                                   control_image=Image.new("RGB", (128, 128)), preloaded_utils=())
    base = dict(color_context=dict(SETTINGS["aurora"]["ctx"]), color_map_image=cmap)
    with pytest.raises(ValueError, match=r"settings\[1\].*control_image"):
        P.paint_with_words_batch([dict(base, control_image=Image.new("RGB", (64, 64))), base], controlnet=net,
                                 preloaded_utils=())
    with pytest.raises(ValueError, match="controlnet is None"):
        P.paint_with_words_batch([dict(base, control_image=Image.new("RGB", (64, 64)))], preloaded_utils=())


def test_control_image_tensor_is_rgb_over_255():
    img = Image.new("RGB", (16, 8), (255, 51, 0))
    t = PL.control_image_tensor(img)
    assert tuple(t.shape) == (1, 3, 8, 16) and t.dtype == torch.float32
    assert torch.equal(t[0, :, 0, 0], torch.tensor([255.0, 51.0, 0.0]) / 255.0) and 0.0 <= t.min() and t.max() <= 1.0


def test_public_signatures_take_the_control_arguments():
    keys = ("controlnet", "control_image", "controlnet_conditioning_scale", "guess_mode", "control_guidance_start",
            "control_guidance_end")
    for fn in (P.paint_with_words, P.paint_with_words_inpaint):
        params = inspect.signature(fn).parameters
        assert all(k in params for k in keys), fn
    params = inspect.signature(P.paint_with_words_batch).parameters
    assert all(k in params for k in ("controlnet", "guess_mode", "control_guidance_start", "control_guidance_end"))
    assert "control_image" in PL.BATCH_SETTING_KEYS and "controlnet_conditioning_scale" in PL.BATCH_SETTING_KEYS
    for cls in (P.PaintWithWord_StableDiffusionPipeline, P.PaintWithWord_StableDiffusionInpaintPipeline):
        assert "controlnet" in inspect.signature(cls.__init__).parameters
        params = inspect.signature(cls.__call__).parameters
        assert all(k in params for k in keys[1:]), cls
    assert P.ControlNetModel is ControlNetModel and P.pww_load_controlnet is pww_load_controlnet


def test_load_controlnet_paths():
    net = pww_load_controlnet("synthetic:tiny", device="cpu", torch_dtype=torch.float32)
    try:
        assert isinstance(net, ControlNetModel) and net.config == UNetConfig.tiny()
        assert net.conv_in.weight.dtype == torch.float32
        with pytest.raises(ValueError, match="model_path"):
            pww_load_controlnet("lllyasviel/sd-controlnet-canny", device="cpu")
    finally:
        P.unpatch_all()


def test_reference_loop_with_the_window_closed_is_the_plain_loop(models):
    """The oracle's own consistency: with no step in the window it is `reference_denoise_loop` exactly."""
    unet, net = models
    sch, conds, unconds, lat = _sampler_inputs(m=1)
    try:
        oracle_loop.patch_with_oracle(unet)
        plain = oracle_loop.reference_denoise_loop(unet, sch, dict(conds[0]), dict(unconds[0]), lat, WF, 7.5)
        closed = reference_controlnet_loop(unet, net, sch, dict(conds[0]), dict(unconds[0]), lat, WF,
                                           torch.rand(1, 3, 64, 64), control_guidance_start=0.9,
                                           control_guidance_end=0.95)
        on = reference_controlnet_loop(unet, net, sch, dict(conds[0]), dict(unconds[0]), lat, WF,
                                       torch.rand(1, 3, 64, 64))
    finally:
        cls = attention_modules(unet)[0].__class__
        if "__call__" in cls.__dict__:
            delattr(cls, "__call__")
    assert torch.equal(plain, closed)
    assert not torch.allclose(plain, on, rtol=3e-2, atol=1e-3)


# ---------------------------------------------------------------------------------------------------------------------
# pww_control_inject_{f16,bf16}: validation before any CUDA call
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name", ["pww_control_inject_f16", "pww_control_inject_bf16"])
def test_control_inject_rejects_bad_arguments_without_gpu(name):
    fn = getattr(_native.lib(), name)
    buf = (ctypes.c_char * 4096)()
    p16 = (ctypes.addressof(buf) + 15) // 16 * 16

    def call(n=2, dst=None, res=None, elems=None, rows=1, count=None):
        k = n if count is None else count
        d = (ctypes.c_void_p * max(k, 1))(*([p16] * k if dst is None else dst))
        r = (ctypes.c_void_p * max(k, 1))(*([p16 + 512] * k if res is None else res))
        e = (ctypes.c_int64 * max(k, 1))(*([16] * k if elems is None else elems))
        return fn(n, d, r, e, rows, None, None)
    assert call(n=0, count=1) == -1
    assert call(n=17) == -1
    assert call(n=-1, count=1) == -1
    assert call(rows=0) == -1
    assert call(rows=-2) == -1
    assert call(elems=[16, 0]) == -1
    assert call(elems=[-8, 16]) == -1
    assert call(elems=[16, 12]) == -1
    assert call(dst=[p16, None]) == -1
    assert call(res=[None, p16]) == -1
    assert call(dst=[p16, p16 + 8]) == -1
    assert call(res=[p16 + 2, p16]) == -1
    assert fn(1, None, None, None, 1, None, None) == -1
