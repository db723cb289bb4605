"""T2I-Adapter units on the CPU: the model's feature shapes at every config, the nearest resize at a ragged latent, the
state-dict round trip and kind inference of `pww_load_adapter`, argument validation of the loader and the sampler, the
guess-scale table, the sampler's per-active-set feature sums, the slow-route UNet with zero features, and
`pww_adapter_residual_*` argument validation (no GPU)."""
import ctypes

import pytest
import torch
import torch.nn.functional as F

import paint_with_words_sd_b200 as P
from oracle import loop as oracle_loop
from paint_with_words_sd_b200 import _native
from paint_with_words_sd_b200 import pipeline as PL
from paint_with_words_sd_b200.adapter import (ADAPTER_GUESS_SCALES, adapter_scales, align_features, build_adapter,
                                              pww_load_adapter, unet_level_sizes)
from paint_with_words_sd_b200.controlnet import build_controlnet
from paint_with_words_sd_b200.unet import UNetConfig, attention_modules, build_unet, combine_control_residuals
from tests.test_multi_controlnet import _imgs, _sampler_inputs

CFG = UNetConfig.tiny()
WF = lambda w, sigma, qk: 0.4 * w * qk.max()     # noqa: E731
KINDS = {"full64": ("full", 64), "full192": ("full", 192), "light": ("light", 192)}
CONFIGS = {"sd15": UNetConfig.sd15, "sd21": UNetConfig.sd21, "tiny": UNetConfig.tiny}


@pytest.mark.parametrize("config", sorted(CONFIGS))
@pytest.mark.parametrize("kind", sorted(KINDS))
def test_feature_shapes_are_the_unet_level_shapes(config, kind):
    cfg = CONFIGS[config]()
    net = build_adapter(cfg, *KINDS[kind])
    with torch.no_grad():
        feats = net(torch.rand(1, 3, 512, 512, generator=torch.manual_seed(0)))
    assert [tuple(f.shape) for f in feats] == [(1, c, h, w) for c, (h, w) in
                                               zip(cfg.block_out_channels, unet_level_sizes(64, 64))]
    assert all(torch.isfinite(f).all() for f in feats)


def test_ragged_latent_features_are_resized_nearest():
    net = build_adapter(CFG, "full", 192)
    with torch.no_grad():
        feats = net(torch.rand(2, 3, 288, 352, generator=torch.manual_seed(1)))
    sizes = unet_level_sizes(36, 44)
    assert sizes == [(36, 44), (18, 22), (9, 11), (5, 6)]
    assert [tuple(f.shape[-2:]) for f in feats] == [(36, 44), (18, 22), (9, 11), (4, 5)]   # the pools round down
    out = align_features(feats, sizes)
    assert [tuple(f.shape[-2:]) for f in out] == sizes
    assert all(a is b for a, b in zip(out[:3], feats[:3]))
    assert torch.equal(out[3], F.interpolate(feats[3], size=(5, 6), mode="nearest"))


@pytest.mark.parametrize("kind", sorted(KINDS))
def test_state_dict_round_trip_infers_the_kind(tmp_path, kind):
    a = build_adapter(CFG, *KINDS[kind], seed=5)
    path = str(tmp_path / "adapter.pth")
    torch.save(a.state_dict(), path)
    b = pww_load_adapter(path, device="cpu", torch_dtype=torch.float32)
    assert (b.kind, b.cin, b.nums_rb, b.ksize, b.channels) == (a.kind, a.cin, a.nums_rb, a.ksize, a.channels)
    sa, sb = a.state_dict(), b.state_dict()
    assert list(sa) == list(sb) and all(torch.equal(sa[k], sb[k]) for k in sa)


def test_synthetic_names():
    for name, (kind, cin) in KINDS.items():
        net = pww_load_adapter(f"synthetic:tiny:{name}", device="cpu")
        assert (net.kind, net.cin, net.channels, next(net.parameters()).dtype) == (kind, cin, CFG.block_out_channels,
                                                                                   torch.float16)
    assert pww_load_adapter("synthetic:sd21:light", device="cpu").channels == (320, 640, 1280, 1280)


def test_unknown_paths_and_state_dicts_raise(tmp_path):
    for bad in ("synthetic:sd15", "synthetic:sd15:style", "synthetic:xl:full64", "adapter.safetensors",
                str(tmp_path / "missing.pth")):
        with pytest.raises(ValueError):
            pww_load_adapter(bad, device="cpu")
    junk = str(tmp_path / "junk.pth")
    torch.save({"foo.weight": torch.zeros(3)}, junk)
    with pytest.raises(ValueError, match="neither a full adapter"):
        pww_load_adapter(junk, device="cpu")
    sd = build_adapter(CFG, "full", 64).state_dict()
    sd["body.3.extra.weight"] = torch.zeros(1)
    torch.save(sd, junk)
    with pytest.raises(ValueError, match="not a full adapter"):
        pww_load_adapter(junk, device="cpu")
    sd = build_adapter(CFG, "full", 64, nums_rb=3).state_dict()
    del sd["body.11.block1.weight"]
    torch.save(sd, junk)
    with pytest.raises(ValueError):
        pww_load_adapter(junk, device="cpu")


def test_guess_scale_table():
    assert ADAPTER_GUESS_SCALES == (0.25, 0.62, 0.825, 1.0)
    t = adapter_scales([0.5, 1.5], True)
    assert tuple(t.shape) == (4, 2) and t.dtype == torch.float32
    want = torch.tensor([[w * s for w in (0.5, 1.5)] for s in ADAPTER_GUESS_SCALES], dtype=torch.float64)
    assert torch.equal(t, want.to(torch.float32))
    assert torch.equal(adapter_scales([0.5, 1.5], False), torch.tensor([[0.5, 1.5, 0.5, 1.5]] * 4))


def test_slow_route_unet_with_zero_features_is_bitwise_the_plain_unet():
    unet = build_unet(CFG, seed=0)
    x = torch.randn(2, 4, 16, 16, generator=torch.manual_seed(2))
    ctx = torch.randn(2, 77, CFG.cross_attention_dim, generator=torch.manual_seed(3))
    zeros = [torch.zeros(2, c, h, w) for c, (h, w) in zip(CFG.block_out_channels, unet_level_sizes(16, 16))]
    with torch.no_grad():
        plain = unet(x, 500, encoder_hidden_states=ctx).sample
        zero = unet(x, 500, encoder_hidden_states=ctx, down_intrablock_additional_residuals=zeros).sample
        half = unet(x, 500, encoder_hidden_states=ctx,
                    down_intrablock_additional_residuals=[torch.ones_like(z[:1]) for z in zeros]).sample
        full = unet(x, 500, encoder_hidden_states=ctx,
                    down_intrablock_additional_residuals=[torch.ones_like(z) for z in zeros]).sample
        with pytest.raises(ValueError, match="3 down_intrablock"):
            unet(x, 500, encoder_hidden_states=ctx, down_intrablock_additional_residuals=zeros[:3])
        with pytest.raises(ValueError, match="adapter feature"):
            unet(x, 500, encoder_hidden_states=ctx, down_intrablock_additional_residuals=zeros[::-1])
    assert torch.equal(zero, plain)
    # one feature row: only the first image changes
    assert torch.equal(half[1], plain[1]) and not torch.equal(half[0], plain[0])
    assert torch.equal(full[0], half[0])


@pytest.fixture(scope="module")
def models():
    unet = build_unet(CFG, seed=0)
    oracle_loop.patch_with_oracle(unet)
    yield unet, build_adapter(CFG, "full", 192, seed=3), build_adapter(CFG, "light", 192, seed=4), \
        build_controlnet(CFG, seed=1)
    cls = attention_modules(unet)[0].__class__
    if "__call__" in cls.__dict__:
        delattr(cls, "__call__")


def test_sampler_sums_the_active_adapters_once_per_active_set(models):
    unet, a, b, net = models
    sch, conds, unconds, lat = _sampler_inputs(m=2)
    imgs = [_imgs(2), _imgs(1)[0], _imgs(1)[0]]
    s = PL.PwWSampler(unet, sch, conds, unconds, lat, WF, controlnet=[a, net, b], control_image=imgs,
                      controlnet_conditioning_scale=[[0.5, 1.5], 0.7, 0.25], control_guidance_start=[0.0, 0.0, 0.5])
    assert s._active_sets == [(True, True, False)] * 2 + [(True, True, True)] * 2
    assert set(s._adapter_sums) == set(s._combine_scales) == {(True, True, False), (True, True, True)}
    assert all(t.shape[0] == 1 for t in s._combine_scales.values())     # the one ControlNet's table
    assert s._hints[0] is None and s._hints[2] is None and tuple(s._hints[1].shape) == (4, 160, 8, 8)
    with torch.no_grad():
        fa = [torch.cat([f, f]) for f in a(torch.cat(imgs[0]))]
        fb = [torch.cat([f, f]) for f in b(torch.cat([imgs[2]] * 2))]
    sa = adapter_scales([0.5, 1.5], False)
    sb = adapter_scales([0.25, 0.25], False)
    assert all(torch.equal(x, y) for x, y in
               zip(s._adapter_sums[(True, True, False)], combine_control_residuals([fa], sa[None])))
    assert all(torch.equal(x, y) for x, y in
               zip(s._adapter_sums[(True, True, True)], combine_control_residuals([fa, fb], torch.stack([sa, sb]))))
    assert [tuple(t.shape) for t in s._adapter_sums[(True, True, True)]] == [(4, 160, 8, 8), (4, 320, 4, 4),
                                                                              (4, 640, 2, 2), (4, 640, 1, 1)]


def test_guess_mode_adapter_routes_to_the_cond_half(models):
    unet, a, _, _ = models
    sch, conds, unconds, lat = _sampler_inputs(m=2)
    s = PL.PwWSampler(unet, sch, conds, unconds, lat, WF, controlnet=a, control_image=_imgs(2),
                      controlnet_conditioning_scale=[0.5, 2.0], guess_mode=True)
    with torch.no_grad():
        fa = a(torch.cat(_imgs(2)))
    got = s._adapter_sums[(True,)]
    assert [t.shape[0] for t in got] == [2] * 4
    want = combine_control_residuals([fa], adapter_scales([0.5, 2.0], True)[None])
    assert all(torch.equal(x, y) for x, y in zip(got, want))


def test_sampler_rejects_bad_adapter_arguments(models):
    unet, a, _, net = models
    sch, conds, unconds, lat = _sampler_inputs()
    with pytest.raises(ValueError, match="block_out_channels"):
        PL.PwWSampler(unet, sch, conds, unconds, lat, WF, controlnet=build_adapter(UNetConfig.sd15()),
                      control_image=_imgs(1)[0])
    with pytest.raises(ValueError, match=r"control_image\[1\] 0 is \(1, 3, 32, 32\)"):
        PL.PwWSampler(unet, sch, conds, unconds, lat, WF, controlnet=[net, a],
                      control_image=[_imgs(1)[0], torch.rand(1, 3, 32, 32)])
    with pytest.raises(ValueError, match="needs a control_image"):
        PL.PwWSampler(unet, sch, conds, unconds, lat, WF, controlnet=a)
    with pytest.raises(ValueError, match="1 to 10"):
        PL.PwWSampler(unet, sch, conds, unconds, lat, WF, controlnet=[a] * 6 + [net] * 5,
                      control_image=_imgs(1) * 11)
    with pytest.raises(TypeError, match="T2IAdapter"):
        PL.PwWSampler(unet, sch, conds, unconds, lat, WF, controlnet=[a, "net"], control_image=_imgs(2))
    with pytest.raises(ValueError, match="an adapter hint"):
        a(torch.rand(1, 3, 60, 64))


def test_public_names():
    assert P.T2IAdapter is not None and P.pww_load_adapter is pww_load_adapter and P.build_adapter is build_adapter


@pytest.mark.parametrize("name", ["pww_adapter_residual_f16", "pww_adapter_residual_bf16"])
def test_adapter_residual_rejects_bad_arguments(name):
    fn = getattr(_native.lib(), name)
    buf = (ctypes.c_char * 8192)()
    p = (ctypes.addressof(buf) + 15) // 16 * 16
    ok = dict(a=p, b=p + 1024, bias=p + 2048, feat=p + 4096, out=p + 1024, rows=4, pixels=2, C=64, feat_rows=2)

    def call(**kw):
        a = {**ok, **kw}
        return fn(a["a"], a["b"], a["bias"], a["feat"], a["out"], a["rows"], a["pixels"], a["C"], a["feat_rows"], None)

    for ptr in ("a", "b", "out"):
        assert call(**{ptr: None}) == -1, f"null {ptr}"
    for ptr in ("a", "b", "bias", "feat", "out"):
        assert call(**{ptr: ok[ptr] + 2}) == -1, f"misaligned {ptr}"
    assert call(feat=None) == -1                            # feat_rows > 0 needs a feature
    for bad in (dict(rows=0), dict(rows=-3), dict(pixels=0), dict(C=0), dict(C=-8), dict(C=12), dict(C=4),
                dict(feat_rows=-1), dict(feat_rows=5)):
        assert call(**bad) == -1, bad
