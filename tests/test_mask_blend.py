"""Masked img2img without a GPU: the sigma' column of the step rows, argument checks of PwWSampler, paint_with_words and
the C entry point, the mask preparation, and self-checks of the CPU reference loop."""
import ctypes
import math

import numpy as np
import pytest
import torch
from PIL import Image

from oracle import mask_blend_loop, rescale_loop
from paint_with_words_sd_b200 import _native
from paint_with_words_sd_b200 import pipeline as PL
from paint_with_words_sd_b200.scheduler import (FORM_COLUMNS, DPMSolverMultistepScheduler,
                                                EulerAncestralDiscreteScheduler, EulerDiscreteScheduler,
                                                LMSDiscreteScheduler)
from tests.fixtures import color_map_image
from tests.test_vpred import _ToyUNet

WF = lambda w, sigma, qk: 0.4 * w * math.log(1 + sigma) * qk.max()   # noqa: E731
KW = dict(beta_start=0.00085, beta_end=0.012, beta_schedule="scaled_linear")
SCHEDULERS = [LMSDiscreteScheduler, EulerDiscreteScheduler, EulerAncestralDiscreteScheduler,
              DPMSolverMultistepScheduler, lambda **kw: DPMSolverMultistepScheduler(**kw, use_karras_sigmas=True)]
IDS = ["lms", "euler", "euler_a", "dpmpp_2m", "dpmpp_2m_karras"]


def _scheduler(cls, steps, prediction_type="epsilon"):
    sch = cls(**KW, prediction_type=prediction_type)
    sch.set_timesteps(steps)
    return sch


def _blend(m, h=8, w=8, seed=0):
    g = torch.Generator().manual_seed(seed)
    return dict(init_latents=torch.randn(m, 4, h, w, generator=g), init_noise=torch.randn(m, 4, h, w, generator=g),
                inpaint_mask=(torch.rand(m, 1, h, w, generator=g) > 0.5).float())


def _sampler(sch, m=1, start=0, **kw):
    """A CPU sampler over m images (the UNet is never called)."""
    g = torch.Generator().manual_seed(0)
    conds = [{"CONTEXT_TENSOR": torch.randn(1, 77, 32, generator=g)} for _ in range(m)]
    unconds = [{"CONTEXT_TENSOR": torch.randn(1, 77, 32, generator=g)} for _ in range(m)]
    return PL.PwWSampler(torch.nn.Linear(1, 1), sch, conds, unconds, torch.zeros(m, 4, 8, 8), WF, 7.5,
                         use_graph=False, timesteps=sch.timesteps[start:], noise_seed=0, **kw)


# ---- the step rows ---------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("cls", SCHEDULERS, ids=IDS)
@pytest.mark.parametrize("start", [0, 4], ids=["full", "img2img_tail"])
@pytest.mark.parametrize("m", [1, 3])
def test_sigma_next_column(cls, start, m):
    steps = 10
    sch = _scheduler(cls, steps)
    plain = _sampler(sch, m, start)
    masked = _sampler(sch, m, start, **_blend(m))
    form_end = plain._form + len(FORM_COLUMNS)
    assert plain._rows.shape == (steps - start, form_end) and masked._rows.shape == (steps - start, form_end + 1)
    # the rows up to the form are today's, with or without a mask
    assert torch.equal(masked._rows[:, :form_end], plain._rows)
    want = torch.tensor([float(sch.sigmas[i + 1]) for i in range(start, steps)], dtype=torch.float32)
    assert torch.equal(masked._rows[:, form_end], want)
    assert float(masked._rows[-1, form_end]) == 0.0
    # sigma' of every step is the sigma of the next row
    assert torch.equal(masked._rows[:-1, form_end], masked._rows[1:, 0])


def test_rows_without_a_mask_are_recomputed_unchanged():
    """Without a mask, the rows are the layout the step kernels have always read, rebuilt here column by column."""
    sch = _scheduler(LMSDiscreteScheduler, 6)
    s = _sampler(sch, 2, 1)
    rows = []
    for i, (t, (alpha, a, b, beta, gamma)) in enumerate(zip(s.timesteps, s.step_forms())):
        si = sch.step_index_of(t)
        sigma = float(sch.sigmas[si])
        gs = [PL.g_of_sigma(f, pr, sch.sigmas[si]) for f, pr in zip(s._fns, s._probed)]
        rows.append([sigma, 1.0 / math.sqrt(sigma * sigma + 1.0), float(t), *beta, *gs, 0.0, 0.0,
                     alpha, a, b, gamma, float(i % s._hist_len), float(i)])
    assert torch.equal(s._rows, torch.tensor(rows, dtype=torch.float32))
    assert s._blend is None


def test_blend_inputs_are_private_contiguous_fp32_copies():
    sch = _scheduler(EulerDiscreteScheduler, 5)
    b = _blend(2)
    b["init_latents"] = b["init_latents"].double().contiguous(memory_format=torch.channels_last)
    s = _sampler(sch, 2, **b)
    for got, want in zip(s._blend, (b["init_latents"], b["init_noise"], b["inpaint_mask"])):
        assert got.dtype == torch.float32 and got.is_contiguous() and torch.equal(got, want.float())
        assert got.data_ptr() != want.data_ptr()


# ---- argument checks ---------------------------------------------------------------------------------------------------
def test_sampler_blend_arguments_are_validated():
    sch = _scheduler(EulerDiscreteScheduler, 5)
    b = _blend(2)
    for drop in b:
        with pytest.raises(ValueError, match="all three or none"):
            _sampler(sch, 2, **{k: v for k, v in b.items() if k != drop})
    bad = {"init_latents": [torch.zeros(1, 4, 8, 8), torch.zeros(2, 4, 8, 16), torch.zeros(2, 3, 8, 8), "x"],
           "init_noise": [torch.zeros(2, 4, 4, 8), torch.zeros(3, 4, 8, 8)],
           "inpaint_mask": [torch.zeros(2, 4, 8, 8), torch.zeros(2, 8, 8), torch.zeros(1, 1, 8, 8)]}
    for name, values in bad.items():
        for v in values:
            with pytest.raises(ValueError, match=name):
                _sampler(sch, 2, **dict(b, **{name: v}))
    for v in (-0.1, 1.5, float("nan")):
        mask = b["inpaint_mask"].clone()
        mask[1, 0, 3, 3] = v
        with pytest.raises(ValueError, match="inpaint_mask"):
            _sampler(sch, 2, **dict(b, inpaint_mask=mask))
    soft = dict(b, inpaint_mask=torch.full((2, 1, 8, 8), 0.25))
    assert _sampler(sch, 2, **soft)._blend is not None


def test_mask_image_needs_init_image_before_any_model_is_loaded(monkeypatch):
    def no_load(*a, **k):
        raise AssertionError("models loaded before the arguments were checked")
    monkeypatch.setattr(PL, "pww_load_tools", no_load)
    with pytest.raises(ValueError, match="mask_image needs an init_image"):
        PL.paint_with_words(color_context={}, color_map_image=color_map_image("aurora", 64), input_prompt="a",
                            mask_image=Image.new("L", (64, 64), 255), device="cpu")


def test_pipeline_call_passes_mask_image(monkeypatch):
    seen = {}

    def fake(**kw):
        seen.update(kw)
        return torch.zeros(1, 4, 8, 8)
    pipe = PL.PaintWithWord_StableDiffusionPipeline.__new__(PL.PaintWithWord_StableDiffusionPipeline)
    pipe.vae = pipe.text_encoder = pipe.tokenizer = None
    pipe.unet = torch.nn.Linear(1, 1)
    pipe.scheduler = _scheduler(LMSDiscreteScheduler, 3)
    monkeypatch.setattr(PL, "paint_with_words", fake)
    mask, init = Image.new("L", (64, 64), 255), Image.new("RGB", (64, 64))
    pipe("a", color_map_image=init, image=init, mask_image=mask, num_inference_steps=3, output_type="latent")
    assert seen["mask_image"] is mask and seen["init_image"] is init
    seen.clear()
    pipe("a", color_map_image=init, num_inference_steps=3, output_type="latent")
    assert seen["mask_image"] is None and "init_image" not in seen


def test_masked_entry_point_validates_without_a_gpu():
    L = _native.lib()
    buf = (ctypes.c_char * 8192)()
    p = (ctypes.addressof(buf) + 15) // 16 * 16
    F16 = _native.PWW_DTYPE_F16

    def upd(eps=p, dt=F16, lat=p, hist=p, hl=4, noise=None, gs=p, beta=p, form=p, phi=None, stats=None, init=p,
            z0=p, mask=p, sn=p, m=2, h=8, w=8):
        return L.pww_sampler_update_masked(eps, dt, 256, 1, 32, 4, lat, hist, hl, noise, gs, beta, form, phi, stats,
                                           init, z0, mask, sn, m, h, w, None)
    for kw in ({"eps": None}, {"lat": None}, {"hist": None}, {"gs": None}, {"beta": None}, {"form": None},
               {"init": None}, {"z0": None}, {"mask": None}, {"sn": None}, {"stats": p}, {"m": 0}, {"h": 0},
               {"w": 0}, {"hl": 0}, {"hl": 5}):
        assert upd(**kw) == -1, kw
    assert upd(dt=3) == -2 and upd(dt=-1) == -2 and upd(dt=3, phi=p, stats=p) == -2


def test_masked_symbol_is_exported():
    assert "pww_sampler_update_masked" in _native.EXPORTS
    assert hasattr(_native.lib(), "pww_sampler_update_masked")
    L = _native.lib()
    assert len(L.pww_sampler_update_masked.argtypes) == len(L.pww_sampler_update.argtypes) + 6


# ---- the mask and the img2img draw -------------------------------------------------------------------------------------
def test_latent_mask_is_binarised_and_nearest():
    arr = np.zeros((96, 64), dtype=np.uint8)
    arr[:, 32:] = 255
    arr[:40, :] = 127            # < 0.5 after / 255: kept
    arr[40:48, :8] = 128         # >= 0.5: repainted
    mask = Image.fromarray(arr, mode="L").resize((32, 48), Image.NEAREST)     # resized to the init image's size
    init = Image.new("RGB", (64, 96))
    got = PL._latent_mask(init, mask, (12, 8), "cpu")
    small = np.array(mask.resize((64, 96), Image.NEAREST)).astype(np.float32) / 255.0 >= 0.5
    want = torch.nn.functional.interpolate(torch.from_numpy(small.astype(np.float32))[None, None], size=(12, 8))[0, 0]
    assert got.shape == (1, 1, 12, 8) and got.dtype == torch.float32
    assert set(got.unique().tolist()) <= {0.0, 1.0} and torch.equal(got[0, 0], want)
    # white = repaint: the right half is 1 below the grey band
    assert got[0, 0, 6:, 4:].eq(1).all() and got[0, 0, 6:, :4].eq(0).all() and got[0, 0, :5].eq(0).all()


def test_img2img_latents_return_the_init_and_its_noise():
    """The img2img draw is the one it was (one global-RNG draw after the VAE encode), and the start latents are the
    returned init latents noised with the returned noise."""
    from paint_with_words_sd_b200.synthetic import IdentityVAE
    sch = _scheduler(LMSDiscreteScheduler, 10)
    img = color_map_image("aurora", 64)
    torch.manual_seed(7)
    lat, ts, init, z = PL._img2img_latents(IdentityVAE(), sch, img, 10, 0.6, "cpu")
    torch.manual_seed(7)
    assert torch.equal(z, torch.randn(init.shape))
    assert torch.equal(ts, sch.timesteps[4:]) and torch.equal(lat, sch.add_noise(init, z, ts[:1]))
    assert torch.equal(init, 0.18215 * IdentityVAE().encode(PL.preprocess(img)).latent_dist.sample().float())


# ---- the reference loop -------------------------------------------------------------------------------------------------
def _loop_inputs(seed=2, h=8, w=8):
    g = torch.Generator().manual_seed(seed)
    cond = {"CONTEXT_TENSOR": torch.randn(1, 77, 32, generator=g)}
    uncond = {"CONTEXT_TENSOR": torch.randn(1, 77, 32, generator=g)}
    init = torch.randn(1, 4, h, w, generator=g)
    z = torch.randn(1, 4, h, w, generator=g)
    return cond, uncond, init, z


@pytest.mark.parametrize("cls", [LMSDiscreteScheduler, EulerDiscreteScheduler, DPMSolverMultistepScheduler])
@pytest.mark.parametrize("phi", [0.0, 0.7])
def test_oracle_with_an_all_ones_mask_is_the_rescale_loop(cls, phi):
    cond, uncond, init, z = _loop_inputs()
    sch = _scheduler(cls, 8)
    ts = sch.timesteps[3:]
    lat = sch.add_noise(init, z, ts[:1])
    ref = rescale_loop.reference_rescale_loop(_ToyUNet(), _scheduler(cls, 8), dict(cond), dict(uncond), lat, WF, 7.5,
                                              guidance_rescale=phi, timesteps=ts)
    got = mask_blend_loop.reference_mask_blend_loop(_ToyUNet(), _scheduler(cls, 8), dict(cond), dict(uncond), lat,
                                                    WF, init, z, torch.ones(1, 1, 8, 8), 7.5, guidance_rescale=phi,
                                                    timesteps=ts)
    assert torch.equal(got, ref)


@pytest.mark.parametrize("cls", [LMSDiscreteScheduler, EulerDiscreteScheduler, DPMSolverMultistepScheduler])
def test_oracle_with_an_all_zeros_mask_ends_at_init(cls):
    cond, uncond, init, z = _loop_inputs()
    sch = _scheduler(cls, 8)
    ts = sch.timesteps[2:]
    lat = sch.add_noise(init, z, ts[:1])
    got = mask_blend_loop.reference_mask_blend_loop(_ToyUNet(), sch, dict(cond), dict(uncond), lat, WF, init, z,
                                                    torch.zeros(1, 1, 8, 8), 7.5, timesteps=ts)
    assert torch.equal(got, init)


def test_oracle_half_mask_keeps_init_outside_and_repaints_inside():
    cond, uncond, init, z = _loop_inputs()
    mask = torch.zeros(1, 1, 8, 8)
    mask[..., 4:] = 1
    sch = _scheduler(EulerDiscreteScheduler, 8)
    ts = sch.timesteps[2:]
    lat = sch.add_noise(init, z, ts[:1])
    got = mask_blend_loop.reference_mask_blend_loop(_ToyUNet(), sch, dict(cond), dict(uncond), lat, WF, init, z, mask,
                                                    7.5, timesteps=ts)
    assert torch.equal(got[..., :4], init[..., :4]) and not torch.allclose(got[..., 4:], init[..., 4:])


def test_noised_init_is_add_noise_at_the_next_timestep():
    _, _, init, z = _loop_inputs()
    for cls in (LMSDiscreteScheduler, lambda **kw: DPMSolverMultistepScheduler(**kw, use_karras_sigmas=True)):
        sch = _scheduler(cls, 6)
        for i in range(6):
            got = mask_blend_loop.noised_init(sch, init, z, i)
            assert torch.equal(got, init + z * sch.sigmas[i + 1])
            if i + 1 < 6:
                assert torch.equal(got, sch.add_noise(init, z, [sch.timesteps[i + 1]]))
        assert torch.equal(mask_blend_loop.noised_init(sch, init, z, 5), init)
