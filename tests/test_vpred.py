"""v-prediction and guidance rescale without a GPU: the step forms of a v-prediction scheduler against its own `step`,
the host v conversion, argument checks, the model's scheduler config, the batch key and the rescale oracle."""
import ctypes
import functools
import inspect
import json
import math

import pytest
import torch

from oracle import loop as oracle_loop
from oracle import rescale_loop
from paint_with_words_sd_b200 import _native, attention
from paint_with_words_sd_b200 import pipeline as PL
from paint_with_words_sd_b200.scheduler import (DPMSolverMultistepScheduler, EulerAncestralDiscreteScheduler,
                                                EulerDiscreteScheduler, LMSDiscreteScheduler, step_form)
from paint_with_words_sd_b200.synthetic import IdentityVAE, RandomTextEncoder, SimpleWordTokenizer
from tests.fixtures import SETTINGS, color_map_image
from tests.test_samplers import SCHEDULERS, _apply_forms

WF = lambda w, sigma, qk: 0.4 * w * math.log(1 + sigma) * qk.max()   # noqa: E731
KW = dict(beta_start=0.00085, beta_end=0.012, beta_schedule="scaled_linear")


def _scheduler(cls, steps, prediction_type="epsilon"):
    sch = cls(**KW, prediction_type=prediction_type)
    sch.set_timesteps(steps)
    return sch


def _sampler(sch, m=1, start=0, **kw):
    """A CPU sampler over m images (the UNet is never called)."""
    g = torch.Generator().manual_seed(0)
    conds = [{"CONTEXT_TENSOR": torch.randn(1, 77, 32, generator=g)} for _ in range(m)]
    unconds = [{"CONTEXT_TENSOR": torch.randn(1, 77, 32, generator=g)} for _ in range(m)]
    return PL.PwWSampler(torch.nn.Linear(1, 1), sch, conds, unconds, torch.zeros(m, 4, 8, 8), WF, 7.5,
                         use_graph=False, timesteps=sch.timesteps[start:], noise_seed=0, **kw)


# ---- step forms ------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name,cls", SCHEDULERS, ids=[n for n, _ in SCHEDULERS])
def test_epsilon_step_forms_are_unchanged(name, cls):
    """The default and an explicit "epsilon" give the forms of a scheduler built without the argument."""
    for steps in (5, 30):
        plain = cls(**KW)
        plain.set_timesteps(steps)
        for sch in (_scheduler(cls, steps), plain):
            assert sch.config["prediction_type"] == "epsilon"
        eps = _scheduler(cls, steps)
        for i in range(steps):
            for first in (True, False):
                assert step_form(eps, i, first) == step_form(plain, i, first), (i, first)
        # q = eps for LMS and the Euler samplers, q = D = x - sigma eps for DPM++ 2M
        _, a, b, _, _ = step_form(eps, 1, False)
        if isinstance(eps, DPMSolverMultistepScheduler):
            assert (a, b) == (1.0, -float(eps.sigmas[1]))
        else:
            assert (a, b) == (0.0, 1.0)


@pytest.mark.parametrize("name,cls", SCHEDULERS, ids=[n for n, _ in SCHEDULERS])
@pytest.mark.parametrize("steps", [5, 20, 30])
@pytest.mark.parametrize("start", ["first", "mid"])
def test_v_step_forms_equal_the_schedulers_v_step(name, cls, steps, start):
    sch = _scheduler(cls, steps, "v_prediction")
    t0 = 0 if start == "first" else steps // 3
    s = _sampler(sch, start=t0)
    forms = s.step_forms()
    n = len(forms)
    g = torch.Generator().manual_seed(steps)
    x0 = torch.randn(1, 4, 8, 8, generator=g, dtype=torch.float64) * 14.6
    v = [torch.randn(1, 4, 8, 8, generator=g, dtype=torch.float64) for _ in range(n)]
    z = [torch.randn(1, 4, 8, 8, generator=g, dtype=torch.float64) for _ in range(n)]
    got = _apply_forms(forms, s._hist_len, x0, v, z)
    ref_sch = _scheduler(cls, steps, "v_prediction")
    x = x0
    for i, t in enumerate(ref_sch.timesteps[t0:]):
        extra = {"noise": z[i]} if isinstance(ref_sch, EulerAncestralDiscreteScheduler) else {}
        x = ref_sch.step(v[i], t, x, **extra).prev_sample
    err = (got - x).abs().max().item() / x.abs().max().item()
    assert err < 1e-6, err
    # the composition rule against the epsilon forms of the same schedule
    eps_forms = _sampler(_scheduler(cls, steps), start=t0).step_forms()
    for i, ((alpha, a, b, beta, gamma), (ea, ea_, eb, ebeta, egamma)) in enumerate(zip(forms, eps_forms)):
        sigma = float(sch.sigmas[sch.step_index_of(s.timesteps[i])])
        assert (alpha, beta, gamma) == (ea, ebeta, egamma)
        assert a == ea_ + eb * sigma / (sigma * sigma + 1.0) and b == eb / math.sqrt(sigma * sigma + 1.0)


@pytest.mark.parametrize("cls", [LMSDiscreteScheduler, EulerDiscreteScheduler, EulerAncestralDiscreteScheduler,
                                 DPMSolverMultistepScheduler])
def test_host_v_step_is_the_diffusers_conversion(cls):
    """pred_original = -sigma/sqrt(sigma^2+1) v + x/(sigma^2+1); eps = (x - pred_original)/sigma; the epsilon step on
    that eps (DPM++ 2M: the step on D = pred_original, which the epsilon scheduler computes from the same eps)."""
    steps = 8
    vs, es = _scheduler(cls, steps, "v_prediction"), _scheduler(cls, steps)
    g = torch.Generator().manual_seed(5)
    x = torch.randn(1, 4, 8, 8, generator=g, dtype=torch.float64) * 10
    for i in range(steps):
        t = vs.timesteps[i]
        sigma = float(vs.sigmas[i])
        v = torch.randn(1, 4, 8, 8, generator=g, dtype=torch.float64)
        z = torch.randn(1, 4, 8, 8, generator=g, dtype=torch.float64)
        pred = -sigma / math.sqrt(sigma ** 2 + 1) * v + x / (sigma ** 2 + 1)
        eps = (x - pred) / sigma
        extra = {"noise": z} if cls is EulerAncestralDiscreteScheduler else {}
        got = vs.step(v, t, x, **extra)
        want = es.step(eps, t, x, **extra)
        assert (got.pred_original_sample - pred).abs().max().item() < 1e-12 * (1 + pred.abs().max().item())
        d = (got.prev_sample - want.prev_sample).abs().max().item()
        assert d < 1e-9 * (1 + want.prev_sample.abs().max().item()), (i, d)
        x = got.prev_sample


def test_v_form_of_dpmpp_2m_final_step_returns_pred_original():
    for karras in (False, True):
        sch = _scheduler(functools.partial(DPMSolverMultistepScheduler, use_karras_sigmas=karras), 5, "v_prediction")
        alpha, a, b, beta, gamma = step_form(sch, 4, False)
        sigma = float(sch.sigmas[4])
        assert (alpha, beta, gamma) == (0.0, [1.0, 0.0, 0.0, 0.0], 0.0)
        assert math.isclose(a, 1 / (sigma ** 2 + 1), rel_tol=1e-12)
        assert math.isclose(b, -sigma / math.sqrt(sigma ** 2 + 1), rel_tol=1e-12)


# ---- argument checks ---------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("cls", [LMSDiscreteScheduler, EulerDiscreteScheduler, EulerAncestralDiscreteScheduler,
                                 DPMSolverMultistepScheduler])
def test_prediction_type_is_validated(cls):
    for bad in ("sample", "v", "", None):
        with pytest.raises(ValueError, match="prediction_type"):
            cls(**KW, prediction_type=bad)
    assert cls(**KW, prediction_type="v_prediction").config["prediction_type"] == "v_prediction"


def test_guidance_rescale_is_validated():
    sch = _scheduler(EulerDiscreteScheduler, 5, "v_prediction")
    for bad in (-0.1, 1.5, float("nan"), float("inf"), [0.5], [0.5, 0.2, 0.1], True, "0.5"):
        with pytest.raises(ValueError, match="guidance_rescale"):
            _sampler(sch, m=2, guidance_rescale=bad)
    s = _sampler(sch, m=2, guidance_rescale=[0.0, 1.0])
    assert s.guidance_rescale == [0.0, 1.0] and s._rescale.tolist() == [0.0, 1.0]
    s = _sampler(sch, m=2, guidance_rescale=0.7)
    assert s._rescale.tolist() == pytest.approx([0.7, 0.7])
    assert _sampler(sch, m=2)._rescale is None and _sampler(sch, m=2, guidance_rescale=[0, 0])._rescale is None


def test_rescale_entry_point_validates_without_a_gpu():
    L = _native.lib()
    buf = (ctypes.c_char * 8192)()
    p = (ctypes.addressof(buf) + 15) // 16 * 16
    F16 = _native.PWW_DTYPE_F16
    upd = lambda eps=p, dt=F16, lat=p, hist=p, hl=4, noise=None, gs=p, beta=p, form=p, phi=p, stats=None, m=2, h=8, \
        w=8: L.pww_sampler_update_rescale(eps, dt, 256, 1, 32, 4, lat, hist, hl, noise, gs, beta, form, phi, stats,  # noqa: E731
                                          m, h, w, None)
    for kw in ({"eps": None}, {"lat": None}, {"hist": None}, {"gs": None}, {"beta": None}, {"form": None},
               {"phi": None}, {"m": 0}, {"h": 0}, {"w": 0}, {"hl": 0}, {"hl": 5}):
        assert upd(**kw) == -1, kw
    assert upd(dt=3) == -2 and upd(dt=-1) == -2


# ---- loading -----------------------------------------------------------------------------------------------------------
def test_scheduler_config_of_a_local_model_decides(tmp_path):
    (tmp_path / "scheduler").mkdir()
    cfg = tmp_path / "scheduler" / "scheduler_config.json"
    cfg.write_text(json.dumps({"_class_name": "DDIMScheduler", "prediction_type": "v_prediction"}))
    assert PL.model_prediction_type(str(tmp_path)) == "v_prediction"
    cfg.write_text(json.dumps({"_class_name": "PNDMScheduler"}))
    assert PL.model_prediction_type(str(tmp_path)) == "epsilon"
    cfg.unlink()
    assert PL.model_prediction_type(str(tmp_path)) == "epsilon"
    assert PL.model_prediction_type("synthetic:sd21") == "epsilon"


def test_load_tools_passes_prediction_type_to_the_scheduler():
    try:
        for p in ("v_prediction", "epsilon", None):
            sch = PL.pww_load_tools("cpu", hf_model_path="synthetic:tiny", prediction_type=p,
                                    scheduler_type=DPMSolverMultistepScheduler)[4]
            assert isinstance(sch, DPMSolverMultistepScheduler) and sch.config["prediction_type"] == (p or "epsilon")
        with pytest.raises(ValueError, match="prediction_type"):
            PL.pww_load_tools("cpu", hf_model_path="synthetic:tiny", prediction_type="sample")
    finally:
        attention.unpatch_all()


def test_pipeline_classes_keep_the_schedulers_prediction_type():
    try:
        vae, unet, enc, tok, sch = PL.pww_load_tools("cpu", hf_model_path="synthetic:tiny",
                                                     prediction_type="v_prediction")
        pipe = PL.PaintWithWord_StableDiffusionPipeline(vae, enc, tok, unet, scheduler=sch)
        assert isinstance(pipe.scheduler, LMSDiscreteScheduler)
        assert pipe.scheduler.config["prediction_type"] == "v_prediction"
        plain = PL.PaintWithWord_StableDiffusionInpaintPipeline(vae, enc, tok, unet)
        assert plain.scheduler.config["prediction_type"] == "epsilon"
    finally:
        attention.unpatch_all()
    for cls in (PL.PaintWithWord_StableDiffusionPipeline, PL.PaintWithWord_StableDiffusionInpaintPipeline):
        assert inspect.signature(cls.__call__).parameters["guidance_rescale"].default == 0.0
    for fn in (PL.paint_with_words, PL.paint_with_words_inpaint, PL.paint_with_words_batch):
        assert inspect.signature(fn).parameters["prediction_type"].default is None
    for fn in (PL.paint_with_words, PL.paint_with_words_inpaint):
        assert inspect.signature(fn).parameters["guidance_rescale"].default == 0.0


# ---- the batch key -----------------------------------------------------------------------------------------------------
class _RecordingSampler:
    """Stands in for PwWSampler: records the guidance rescale each sampler gets."""
    runs = []

    def __init__(self, unet, scheduler, conds, unconds, latents, weight_function, guidance_scale, **kw):
        self.latents = latents
        _RecordingSampler.runs.append(dict(m=len(conds), scales=list(guidance_scale), rescale=kw["guidance_rescale"]))

    def run(self):
        return self.latents


def test_batch_takes_guidance_rescale_per_entry(monkeypatch):
    assert "guidance_rescale" in PL.BATCH_SETTING_KEYS
    assert PL._batch_settings([{"color_map_image": color_map_image("aurora", 64)}])[0]["guidance_rescale"] == 0.0
    monkeypatch.setattr(PL, "PwWSampler", _RecordingSampler)
    _RecordingSampler.runs = []

    class _UNet:
        in_channels = 4
    sch = LMSDiscreteScheduler(**KW, prediction_type="v_prediction")
    tools = (IdentityVAE(), _UNet(), RandomTextEncoder(32), SimpleWordTokenizer(), sch)
    a = SETTINGS["aurora"]
    base = dict(color_context=dict(a["ctx"]), color_map_image=color_map_image("aurora", 64), input_prompt=a["prompt"])
    entries = [dict(base, seed=0, guidance_rescale=0.7), dict(base, seed=1), dict(base, seed=2, guidance_rescale=0.3)]
    PL.paint_with_words_batch(entries, num_inference_steps=3, device="cpu", preloaded_utils=tools, return_latents=True)
    assert [(r["m"], r["rescale"]) for r in _RecordingSampler.runs] == [(3, [0.7, 0.0, 0.3])]


# ---- the rescale oracle --------------------------------------------------------------------------------------------------
class _Out:
    def __init__(self, sample):
        self.sample = sample


class _ToyUNet(torch.nn.Module):
    """A deterministic stand-in UNet whose output depends on the input, the timestep and the context dict."""

    def forward(self, x, t, encoder_hidden_states=None):
        bias = float(encoder_hidden_states["CONTEXT_TENSOR"].mean())
        return _Out(torch.tanh(x * 0.7 + bias) * (1 + float(t) / 1000))


@pytest.mark.parametrize("cls", [LMSDiscreteScheduler, EulerDiscreteScheduler, DPMSolverMultistepScheduler])
@pytest.mark.parametrize("prediction_type", ["epsilon", "v_prediction"])
def test_rescale_oracle_is_the_reference_loop_at_zero(cls, prediction_type):
    g = torch.Generator().manual_seed(2)
    cond = {"CONTEXT_TENSOR": torch.randn(1, 77, 32, generator=g)}
    uncond = {"CONTEXT_TENSOR": torch.randn(1, 77, 32, generator=g)}
    lat = torch.randn(1, 4, 8, 8, generator=g) * 14.6
    runs = []
    for loop in (oracle_loop.reference_denoise_loop, rescale_loop.reference_rescale_loop):
        runs.append(loop(_ToyUNet(), _scheduler(cls, 6, prediction_type), dict(cond), dict(uncond), lat, WF, 7.5))
    assert torch.equal(runs[0], runs[1])
    rescaled = rescale_loop.reference_rescale_loop(_ToyUNet(), _scheduler(cls, 6, prediction_type), dict(cond),
                                                   dict(uncond), lat, WF, 7.5, guidance_rescale=0.7)
    assert torch.isfinite(rescaled).all() and not torch.equal(rescaled, runs[0])


def test_rescale_noise_cfg_matches_its_definition():
    g = torch.Generator().manual_seed(1)
    text = torch.randn(3, 4, 8, 8, generator=g, dtype=torch.float64)
    cfg = torch.randn(3, 4, 8, 8, generator=g, dtype=torch.float64) * 3
    out = rescale_loop.rescale_noise_cfg(cfg, text, 0.7)
    for i in range(3):
        k = 0.7 * float(text[i].std()) / float(cfg[i].std()) + 0.3
        assert torch.allclose(out[i], k * cfg[i], rtol=1e-12, atol=1e-12)
        assert math.isclose(float(out[i].std()), k * float(cfg[i].std()), rel_tol=1e-12)
