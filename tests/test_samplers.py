"""Euler, Euler ancestral and DPM++ 2M without a GPU: sigma schedules, the step-form tables the sampler kernel consumes
against each scheduler's own `step`, the point-mass trajectory, the noise rule, error cases and the argument checks of
the two sampler entry points."""
import ctypes
import functools
import math

import numpy as np
import pytest
import torch

from paint_with_words_sd_b200 import _native
from paint_with_words_sd_b200 import pipeline as PL
from paint_with_words_sd_b200.scheduler import (DPMSolverMultistepScheduler, EulerAncestralDiscreteScheduler,
                                                EulerDiscreteScheduler, LMSDiscreteScheduler, karras_sigmas,
                                                sigma_to_t)

WF = lambda w, sigma, qk: 0.4 * w * math.log(1 + sigma) * qk.max()   # noqa: E731
KW = dict(beta_start=0.00085, beta_end=0.012, beta_schedule="scaled_linear")

SCHEDULERS = [
    ("lms", LMSDiscreteScheduler),
    ("euler", EulerDiscreteScheduler),
    ("euler_karras", functools.partial(EulerDiscreteScheduler, use_karras_sigmas=True)),
    ("euler_a", EulerAncestralDiscreteScheduler),
    ("euler_a_karras", functools.partial(EulerAncestralDiscreteScheduler, use_karras_sigmas=True)),
    ("dpmpp_2m", DPMSolverMultistepScheduler),
    ("dpmpp_2m_karras", functools.partial(DPMSolverMultistepScheduler, use_karras_sigmas=True)),
]


def _scheduler(cls, steps):
    sch = cls(**KW)
    sch.set_timesteps(steps)
    return sch


def _sampler(sch, m=1, start=0, noise_seed=0, size=8):
    """A CPU sampler over m images (the UNet is never called)."""
    g = torch.Generator().manual_seed(0)
    conds = [{"CONTEXT_TENSOR": torch.randn(1, 77, 32, generator=g)} for _ in range(m)]
    unconds = [{"CONTEXT_TENSOR": torch.randn(1, 77, 32, generator=g)} for _ in range(m)]
    return PL.PwWSampler(torch.nn.Linear(1, 1), sch, conds, unconds, torch.zeros(m, 4, size, size), WF, 7.5,
                         use_graph=False, timesteps=sch.timesteps[start:], noise_seed=noise_seed)


# ---- sigma schedules ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("steps", [5, 20, 30])
def test_karras_sigmas_follow_the_closed_form(steps):
    sch = _scheduler(functools.partial(DPMSolverMultistepScheduler, use_karras_sigmas=True), steps)
    ac = sch.alphas_cumprod.double().numpy()
    train = ((1 - ac) / ac) ** 0.5
    smin, smax = float(np.float32(train[0])), float(np.float32(train[-1]))
    i = np.arange(steps)
    want = (smax ** (1 / 7) + i / (steps - 1) * (smin ** (1 / 7) - smax ** (1 / 7))) ** 7
    sig = sch.sigmas.double().numpy()
    assert sig.shape == (steps + 1,) and sig[-1] == 0
    np.testing.assert_allclose(sig[:-1], want, rtol=1e-6)
    assert np.all(np.diff(sig) < 0)
    # fractional timesteps: interpolating the training log-sigmas at t gives sigma back
    log_train = np.log(sch._lms._train_sigmas())
    t = sch.timesteps.numpy()
    assert np.all(np.diff(t) < 0) and not np.all(t == np.round(t))
    back = np.exp(np.interp(t, np.arange(len(log_train)), log_train))
    np.testing.assert_allclose(back, sig[:-1], rtol=1e-5)
    assert abs(sigma_to_t(float(sig[3]), log_train) - t[3]) < 1e-4      # sig is the fp32-rounded sigma
    np.testing.assert_allclose(karras_sigmas(smin, smax, steps), want, rtol=1e-12)


@pytest.mark.parametrize("cls", [EulerDiscreteScheduler, EulerAncestralDiscreteScheduler, DPMSolverMultistepScheduler])
def test_without_karras_the_schedule_is_lms(cls):
    for steps in (5, 30):
        a, b = _scheduler(cls, steps), _scheduler(LMSDiscreteScheduler, steps)
        assert torch.equal(a.sigmas, b.sigmas) and torch.equal(a.timesteps, b.timesteps)
        assert float(a.init_noise_sigma) == float(b.init_noise_sigma)
        x = torch.randn(1, 4, 8, 8)
        t = a.timesteps[2]
        assert torch.equal(a.scale_model_input(x, t), b.scale_model_input(x, t))
        assert torch.equal(a.add_noise(x, x, t[None]), b.add_noise(x, x, t[None]))


# ---- the step form against each scheduler's own step ----------------------------------------------------------------
def _apply_forms(forms, hist_len, x, eps, z):
    """The kernel's step form in float64 over the whole run."""
    ring = [torch.zeros_like(x) for _ in range(hist_len)]
    for i, (alpha, a, b, beta, gamma) in enumerate(forms):
        slot = i % hist_len
        q = a * x + b * eps[i]
        ring[slot] = q
        s = beta[0] * q
        for k in range(1, hist_len):
            s = s + beta[k] * ring[(slot - k) % hist_len]
        x = alpha * x + s + gamma * z[i]
    return x


@pytest.mark.parametrize("name,cls", SCHEDULERS, ids=[n for n, _ in SCHEDULERS])
@pytest.mark.parametrize("steps", [5, 20, 30])
@pytest.mark.parametrize("start", ["first", "mid"])
def test_step_form_tables_equal_the_schedulers_step(name, cls, steps, start):
    sch = _scheduler(cls, steps)
    t0 = 0 if start == "first" else steps // 3
    s = _sampler(sch, start=t0)
    forms = s.step_forms()
    n = len(forms)
    g = torch.Generator().manual_seed(steps)
    x0 = torch.randn(1, 4, 8, 8, generator=g, dtype=torch.float64) * 14.6
    eps = [torch.randn(1, 4, 8, 8, generator=g, dtype=torch.float64) for _ in range(n)]
    z = [torch.randn(1, 4, 8, 8, generator=g, dtype=torch.float64) for _ in range(n)]
    got = _apply_forms(forms, s._hist_len, x0, eps, z)
    ref_sch = _scheduler(cls, steps)
    x = x0
    for i, t in enumerate(ref_sch.timesteps[t0:]):
        extra = {"noise": z[i]} if isinstance(ref_sch, EulerAncestralDiscreteScheduler) else {}
        x = ref_sch.step(eps[i], t, x, **extra).prev_sample
    err = (got - x).abs().max().item() / x.abs().max().item()
    assert err < 1e-6, err
    # the uploaded fp32 rows are these float64 values rounded, plus the history slot and the noise row
    rows = s._rows.double()
    for i, (alpha, a, b, beta, gamma) in enumerate(forms):
        want = torch.tensor([*beta], dtype=torch.float32).double()
        assert torch.equal(rows[i, 3:7], want)
        form = torch.tensor([alpha, a, b, gamma, i % s._hist_len, i], dtype=torch.float32).double()
        assert torch.equal(rows[i, -6:], form), i


def test_dpmpp_2m_final_step_returns_the_denoised_sample():
    sch = _scheduler(DPMSolverMultistepScheduler, 5)
    alpha, a, b, beta, gamma = _sampler(sch).step_forms()[-1]
    assert (alpha, a, beta, gamma) == (0.0, 1.0, [1.0, 0.0, 0.0, 0.0], 0.0) and b == -float(sch.sigmas[4])
    x, e = torch.randn(1, 4, 8, 8, dtype=torch.float64), torch.randn(1, 4, 8, 8, dtype=torch.float64)
    out = sch.step(e, sch.timesteps[4], x).prev_sample
    assert torch.isfinite(out).all() and torch.equal(out, x - float(sch.sigmas[4]) * e)


@pytest.mark.parametrize("name,cls", SCHEDULERS, ids=[n for n, _ in SCHEDULERS])
def test_point_mass_trajectory_ends_at_x0(name, cls):
    """With the exact denoiser of a point mass at x0, eps = (x - x0) / sigma, every sampler lands on x0.  The last step
    (to sigma' = 0) lands there whatever came before, so the deterministic samplers are also held to the exact
    trajectory x_i = x0 + sigma_i (x_T - x0) / sigma_T at every step; the step form equals `step` (above)."""
    for steps in (5, 20):
        sch = _scheduler(cls, steps)
        g = torch.Generator().manual_seed(1)
        x0 = torch.randn(1, 4, 8, 8, generator=g, dtype=torch.float64)
        xT = x0 + float(sch.sigmas[0]) * torch.randn(1, 4, 8, 8, generator=g, dtype=torch.float64)
        ancestral = isinstance(sch, EulerAncestralDiscreteScheduler)
        x = xT
        for i, t in enumerate(sch.timesteps):
            sigma = float(sch.sigmas[i])
            extra = {"noise": torch.randn(x.shape, generator=g, dtype=torch.float64)} if ancestral else {}
            x = sch.step((x - x0) / sigma, t, x, **extra).prev_sample
            if not ancestral:
                exact = x0 + float(sch.sigmas[i + 1]) / float(sch.sigmas[0]) * (xT - x0)
                assert (x - exact).abs().max().item() < 1e-7 * xT.abs().max().item(), (name, steps, i)
        assert (x - x0).abs().max().item() < 1e-7, name      # LMS: coefficients integrated by quadrature


# ---- layouts and shapes the sampler accepts -------------------------------------------------------------------------
def test_sampler_keeps_a_contiguous_copy_of_channels_last_latents():
    sch = _scheduler(EulerDiscreteScheduler, 5)
    conds, unconds = [{"CONTEXT_TENSOR": torch.randn(1, 77, 32)} for _ in range(2)], \
        [{"CONTEXT_TENSOR": torch.randn(1, 77, 32)} for _ in range(2)]
    lat = torch.randn(2, 4, 8, 8).contiguous(memory_format=torch.channels_last)
    extra = torch.randn(2, 5, 8, 8).contiguous(memory_format=torch.channels_last)
    s = PL.PwWSampler(torch.nn.Linear(1, 1), sch, conds, unconds, lat, WF, extra_input=extra, use_graph=False)
    assert s.latents.is_contiguous() and torch.equal(s.latents, lat) and s.latents.data_ptr() != lat.data_ptr()
    assert s.extra_input.is_contiguous() and torch.equal(s.extra_input, extra)
    half = torch.randn(2, 4, 8, 8, dtype=torch.float16)[:, :, :, ::1].transpose(2, 3)
    s = PL.PwWSampler(torch.nn.Linear(1, 1), sch, conds, unconds, half, WF, use_graph=False)
    assert s.latents.dtype == torch.float32 and s.latents.is_contiguous() and torch.equal(s.latents, half.float())


@pytest.mark.parametrize("lat_shape,extra_shape", [
    ((1, 4, 8, 8), None),            # one latent for two images
    ((3, 4, 8, 8), None),
    ((2, 9, 8, 8), None),            # inpaint channels belong in extra_input
    ((2, 4, 8), None),
    ((2, 4, 8, 8), (1, 5, 8, 8)),
    ((2, 4, 8, 8), (2, 4, 8, 8)),
    ((2, 4, 8, 8), (2, 5, 4, 4)),
])
def test_sampler_rejects_latents_or_extra_input_of_the_wrong_shape(lat_shape, extra_shape):
    sch = _scheduler(EulerDiscreteScheduler, 5)
    conds, unconds = [{"CONTEXT_TENSOR": torch.randn(1, 77, 32)} for _ in range(2)], \
        [{"CONTEXT_TENSOR": torch.randn(1, 77, 32)} for _ in range(2)]
    extra = None if extra_shape is None else torch.zeros(extra_shape)
    with pytest.raises(ValueError, match="extra_input" if extra_shape else "latents"):
        PL.PwWSampler(torch.nn.Linear(1, 1), sch, conds, unconds, torch.zeros(lat_shape), WF, extra_input=extra,
                      use_graph=False)


# ---- errors and the noise rule --------------------------------------------------------------------------------------
def test_unknown_scheduler_is_a_type_error():
    class PNDMScheduler:
        timesteps = torch.arange(3)
    with pytest.raises(TypeError, match="EulerAncestralDiscreteScheduler"):
        PL.PwWSampler(torch.nn.Linear(1, 1), PNDMScheduler(), [{}], [{}], torch.zeros(1, 4, 8, 8), WF)


def test_ancestral_sampler_needs_one_noise_seed_per_image():
    sch = _scheduler(EulerAncestralDiscreteScheduler, 5)
    with pytest.raises(ValueError, match="noise_seed"):
        _sampler(sch, noise_seed=None)
    with pytest.raises(ValueError, match="noise_seed"):
        _sampler(sch, m=2, noise_seed=[1, 2, 3])
    assert _sampler(_scheduler(EulerDiscreteScheduler, 5), noise_seed=None)._noise is None


def test_ancestral_noise_is_draws_one_to_n_of_each_seed():
    sch = _scheduler(EulerAncestralDiscreteScheduler, 6)
    s = _sampler(sch, m=2, start=2, noise_seed=[11, 5])
    assert s._noise.shape == (4, 2, 4, 8, 8)
    for i, seed in enumerate((11, 5)):
        g = torch.manual_seed(seed)
        first = torch.randn(1, 4, 8, 8, generator=g)
        draws = [torch.randn(1, 4, 8, 8, generator=g) for _ in range(4)]
        for k in range(4):
            assert torch.equal(s._noise[k, i], draws[k][0]), (i, k)
        assert not torch.equal(s._noise[0, i], first[0])
    # one seed for every image, and per-image noise does not depend on the batch
    solo = _sampler(_scheduler(EulerAncestralDiscreteScheduler, 6), start=2, noise_seed=5)
    assert torch.equal(solo._noise[:, 0], s._noise[:, 1])


def test_lms_step_table_is_unchanged():
    """The LMS rows are [sigma, 1/sqrt(sigma^2+1), t, c0..c3, G...] as before, with the identity step form."""
    for steps, start in ((5, 0), (30, 0), (30, 12)):
        sch = _scheduler(LMSDiscreteScheduler, steps)
        s = _sampler(sch, start=start)
        rows = []
        for t in s.timesteps:
            si = sch.step_index_of(t)
            sigma = float(sch.sigmas[si])
            coeffs = (list(sch._coeffs[si]) + [0.0] * 4)[:4]
            rows.append([sigma, 1.0 / math.sqrt(sigma * sigma + 1.0), float(t), *coeffs,
                         PL.g_of_sigma(WF, s._probed[0], sch.sigmas[si])])
        assert torch.equal(s._table, torch.tensor(rows, dtype=torch.float32))
        n = len(s.timesteps)
        form = torch.tensor([[1.0, 0.0, 1.0, 0.0, i % 4, i] for i in range(n)], dtype=torch.float32)
        assert torch.equal(s._rows[:, -6:], form) and s._hist_len == 4 and s._noise is None
        assert s._params.numel() == 7 + 2 + 6 and s._ctx["G_SIGMA"].numel() == 2


# ---- argument checks of the C entry points --------------------------------------------------------------------------
def test_sampler_entry_points_validate_without_a_gpu():
    L = _native.lib()
    buf = (ctypes.c_char * 8192)()
    p = (ctypes.addressof(buf) + 15) // 16 * 16
    F32, F16 = _native.PWW_DTYPE_F32, _native.PWW_DTYPE_F16
    inp = lambda lat=p, scale=p, extra=None, out=p, dt=F16, m=1, c=4, h=8, w=8: L.pww_sampler_input(  # noqa: E731
        lat, scale, extra, out, dt, m, c, h, w, None)
    assert inp(lat=None) == -1 and inp(scale=None) == -1 and inp(out=None) == -1
    assert inp(m=0) == -1 and inp(h=0) == -1 and inp(w=-2) == -1
    assert inp(c=5) == -1 and inp(c=9) == -1 and inp(extra=p) == -1        # 9 channels need `extra`, 4 take none
    assert inp(dt=2) == -2 and inp(dt=-1, c=9, extra=p) == -2
    upd = lambda eps=p, dt=F16, lat=p, hist=p, hl=4, noise=None, gs=p, beta=p, form=p, m=2, h=8, w=8: \
        L.pww_sampler_update(eps, dt, 256, 1, 32, 4, lat, hist, hl, noise, gs, beta, form, m, h, w, None)  # noqa: E731
    for kw in ({"eps": None}, {"lat": None}, {"hist": None}, {"gs": None}, {"beta": None}, {"form": None},
               {"m": 0}, {"h": 0}, {"w": 0}, {"hl": 0}, {"hl": 5}):
        assert upd(**kw) == -1, kw
    assert upd(dt=3) == -2 and upd(dt=-1) == -2
    assert L.pww_status_str(-2).startswith(b"unsupported")
