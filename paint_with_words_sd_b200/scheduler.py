"""Minimal LMS discrete scheduler with the diffusers-0.10.0 `LMSDiscreteScheduler` call surface used at
paint_with_words.py:197-202, 431-476, 506 and paint_with_words_inpaint.py:180-197, 266.

diffusers is a third-party dependency that is not vendored in the reference (requirements.txt:1
pins 0.10.0) and is not installed here, so the published algorithm is restated: scaled-linear betas
0.00085..0.012 over 1000 train steps, Karras-style sigmas = sqrt((1-abar)/abar) interpolated at
linspace(0,999,n)[::-1] with a trailing 0, epsilon prediction, order-4 linear multistep with
coefficients from scipy.integrate.quad(epsrel=1e-4).

GPU-first change: the multistep coefficients of every step are integrated once in `set_timesteps`
(the stock implementation calls scipy.quad on the host inside every `step`, stalling the stream), and
`step_index_of` avoids the `.nonzero().item()` device sync of paint_with_words.py:473.

Euler, Euler ancestral and DPM++ 2M (below) are restated the same way from their published definitions (Karras et al.
2022; k-diffusion's `sample_euler_ancestral` / `sample_dpmpp_2m`; Lu et al. 2022), on the LMS schedule or the Karras
schedule.  `step_form` writes any of the four as the one linear update the sampler kernel runs.

Every scheduler takes `prediction_type`: "epsilon" (the model predicts the noise) or "v_prediction" (the SD2.x 768
models: v = sqrt(abar) eps - sqrt(1 - abar) x0, Salimans & Ho 2022), converted in sigma space as diffusers' schedulers
do: x0 = -sigma/sqrt(sigma^2+1) v + x/(sigma^2+1), eps = (x - x0)/sigma.
"""
from __future__ import annotations

import math
from typing import List, Optional

import numpy as np
import torch
from scipy import integrate


PREDICTION_TYPES = ("epsilon", "v_prediction")


def check_prediction_type(prediction_type: str) -> None:
    if prediction_type not in PREDICTION_TYPES:
        raise ValueError(f"prediction_type must be one of {PREDICTION_TYPES}, got {prediction_type!r}")


def predicted_original(prediction_type: str, model_output, sample, sigma: float):
    """x0 from the model output at noise level sigma: x - sigma eps, or -sigma/sqrt(sigma^2+1) v + x/(sigma^2+1)."""
    if prediction_type == "epsilon":
        return sample - sigma * model_output
    return model_output * (-sigma / (sigma ** 2 + 1) ** 0.5) + (sample / (sigma ** 2 + 1))


def predicted_eps(prediction_type: str, model_output, sample, sigma: float):
    """eps from the model output: the output itself, or (x - x0)/sigma for a v output."""
    if prediction_type == "epsilon":
        return model_output
    return (sample - predicted_original(prediction_type, model_output, sample, sigma)) / sigma


class _StepOutput:
    def __init__(self, prev_sample, pred_original_sample):
        self.prev_sample = prev_sample
        self.pred_original_sample = pred_original_sample


class LMSDiscreteScheduler:
    order = 1

    def __init__(self, beta_start: float = 0.0001, beta_end: float = 0.02, beta_schedule: str = "linear",
                 num_train_timesteps: int = 1000, prediction_type: str = "epsilon"):
        check_prediction_type(prediction_type)
        if beta_schedule == "linear":
            betas = np.linspace(beta_start, beta_end, num_train_timesteps, dtype=np.float32)
        elif beta_schedule == "scaled_linear":
            betas = np.linspace(beta_start ** 0.5, beta_end ** 0.5, num_train_timesteps, dtype=np.float32) ** 2
        else:
            raise NotImplementedError(beta_schedule)
        self.config = {"num_train_timesteps": num_train_timesteps, "beta_start": beta_start,
                       "beta_end": beta_end, "beta_schedule": beta_schedule, "prediction_type": prediction_type}
        self.betas = torch.from_numpy(betas)
        self.alphas_cumprod = torch.cumprod(1.0 - self.betas, dim=0)
        sig = self._train_sigmas()
        self.sigmas = torch.from_numpy(np.concatenate([sig[::-1], [0.0]]).astype(np.float32))
        self.init_noise_sigma = self.sigmas.max()
        self.timesteps = torch.from_numpy(
            np.linspace(0, num_train_timesteps - 1, num_train_timesteps, dtype=float)[::-1].copy())
        self.num_inference_steps: Optional[int] = None
        self.derivatives: List[torch.Tensor] = []
        self._coeffs: Optional[List[List[float]]] = None
        self._t_list: List[float] = self.timesteps.tolist()

    def _train_sigmas(self) -> np.ndarray:
        ac = self.alphas_cumprod.numpy()
        return np.array(((1 - ac) / ac) ** 0.5)

    # ---- schedule ------------------------------------------------------------------------
    def set_timesteps(self, num_inference_steps: int, device=None):
        self.num_inference_steps = num_inference_steps
        n_train = self.config["num_train_timesteps"]
        timesteps = np.linspace(0, n_train - 1, num_inference_steps, dtype=float)[::-1].copy()
        sig = self._train_sigmas()
        sig = np.interp(timesteps, np.arange(0, len(sig)), sig)
        sig = np.concatenate([sig, [0.0]]).astype(np.float32)
        self.sigmas = torch.from_numpy(sig)            # host copy: sigma is host scalar math (pww.py:402-405)
        self.timesteps = torch.from_numpy(timesteps).to(device=device)
        self._t_list = timesteps.tolist()
        self.derivatives = []
        self._coeffs = [self._lms_coeffs(i, min(i + 1, 4)) for i in range(num_inference_steps)]

    def get_lms_coefficient(self, order: int, t: int, current_order: int) -> float:
        sig = self.sigmas

        def lms_derivative(tau):
            prod = 1.0
            for k in range(order):
                if current_order == k:
                    continue
                prod *= (tau - sig[t - k]) / (sig[t - current_order] - sig[t - k])
            return prod

        return integrate.quad(lms_derivative, sig[t], sig[t + 1], epsrel=1e-4)[0]

    def _lms_coeffs(self, step_index: int, order: int) -> List[float]:
        return [float(self.get_lms_coefficient(order, step_index, o)) for o in range(order)]

    def step_index_of(self, timestep) -> int:
        """Host lookup of the schedule position of `timestep` (no device sync)."""
        t = float(timestep)
        for i, v in enumerate(self._t_list):
            if v == t:
                return i
        raise ValueError(f"timestep {t} is not on the schedule")

    # ---- per-step ------------------------------------------------------------------------
    def scale_model_input(self, sample: torch.Tensor, timestep) -> torch.Tensor:
        sigma = float(self.sigmas[self.step_index_of(timestep)])
        return sample / ((sigma ** 2 + 1) ** 0.5)

    def step(self, model_output: torch.Tensor, timestep, sample: torch.Tensor, order: int = 4):
        i = self.step_index_of(timestep)
        sigma = float(self.sigmas[i])
        pred_original_sample = predicted_original(self.config["prediction_type"], model_output, sample, sigma)
        derivative = (sample - pred_original_sample) / sigma
        self.derivatives.append(derivative)
        if len(self.derivatives) > order:
            self.derivatives.pop(0)
        order = min(i + 1, order)
        coeffs = self._coeffs[i][:order] if (self._coeffs is not None and order == min(i + 1, 4)) \
            else self._lms_coeffs(i, order)
        prev_sample = sample + sum(c * d for c, d in zip(coeffs, reversed(self.derivatives)))
        return _StepOutput(prev_sample, pred_original_sample)

    def add_noise(self, original_samples: torch.Tensor, noise: torch.Tensor, timesteps) -> torch.Tensor:
        idx = [self.step_index_of(t) for t in timesteps]
        sigma = self.sigmas[idx].flatten().to(original_samples.device, original_samples.dtype)
        while sigma.dim() < original_samples.dim():
            sigma = sigma.unsqueeze(-1)
        return original_samples + noise * sigma


# ---------------------------------------------------------------------------------------------------------------------
# Euler, Euler ancestral and DPM++ 2M (sigma space)
# ---------------------------------------------------------------------------------------------------------------------
def karras_sigmas(sigma_min: float, sigma_max: float, n: int, rho: float = 7.0) -> np.ndarray:
    """Karras et al. 2022, eq. (5): sigma_i = (max^(1/rho) + i/(n-1) (min^(1/rho) - max^(1/rho)))^rho, i = 0 .. n-1."""
    ramp = np.linspace(0, 1, n)
    lo, hi = sigma_min ** (1 / rho), sigma_max ** (1 / rho)
    return (hi + ramp * (lo - hi)) ** rho


def sigma_to_t(sigma: float, log_sigmas: np.ndarray) -> float:
    """Fractional train timestep of `sigma`: linear interpolation in log sigma between the two bracketing training sigmas
    (diffusers' `_sigma_to_t`); `log_sigmas` ascends with t."""
    log_sigma = np.log(sigma)
    low = min(int(np.cumsum(log_sigma - log_sigmas >= 0).argmax()), log_sigmas.shape[0] - 2)
    w = float(np.clip((log_sigmas[low] - log_sigma) / (log_sigmas[low] - log_sigmas[low + 1]), 0, 1))
    return (1 - w) * low + w * (low + 1)


class _SigmaScheduler:
    """Shared schedule of the sigma-space samplers: the LMS schedule (sigmas interpolated at linspace(0, 999, n)[::-1],
    trailing 0) or, with `use_karras_sigmas`, the Karras schedule between the training sigma_min and sigma_max with
    fractional timesteps.  Subclasses define `step`."""
    order = 1

    def __init__(self, beta_start: float = 0.0001, beta_end: float = 0.02, beta_schedule: str = "linear",
                 num_train_timesteps: int = 1000, use_karras_sigmas: bool = False, prediction_type: str = "epsilon"):
        self._lms = LMSDiscreteScheduler(beta_start, beta_end, beta_schedule, num_train_timesteps, prediction_type)
        self.config = dict(self._lms.config, use_karras_sigmas=use_karras_sigmas)
        self.use_karras_sigmas = use_karras_sigmas
        self.betas, self.alphas_cumprod = self._lms.betas, self._lms.alphas_cumprod
        self.sigmas, self.timesteps = self._lms.sigmas, self._lms.timesteps
        self.init_noise_sigma = self._lms.init_noise_sigma
        self.num_inference_steps: Optional[int] = None
        self._t_list: List[float] = self.timesteps.tolist()
        self._reset()

    def _reset(self):
        pass

    def set_timesteps(self, num_inference_steps: int, device=None):
        self.num_inference_steps = num_inference_steps
        if not self.use_karras_sigmas:
            self._lms.set_timesteps(num_inference_steps)
            sig, timesteps = self._lms.sigmas, np.array(self._lms._t_list)
        else:
            train = self._lms._train_sigmas()
            s = karras_sigmas(float(train[0]), float(train[-1]), num_inference_steps)
            log_sigmas = np.log(train)
            timesteps = np.array([sigma_to_t(x, log_sigmas) for x in s])
            sig = torch.from_numpy(np.concatenate([s, [0.0]]).astype(np.float32))
        self.sigmas = sig
        self.timesteps = torch.from_numpy(timesteps).to(device=device)
        self._t_list = timesteps.tolist()
        self._reset()

    def step_index_of(self, timestep) -> int:
        """Host lookup of the schedule position of `timestep` (no device sync)."""
        t = float(timestep)
        for i, v in enumerate(self._t_list):
            if v == t:
                return i
        raise ValueError(f"timestep {t} is not on the schedule")

    def scale_model_input(self, sample: torch.Tensor, timestep) -> torch.Tensor:
        sigma = float(self.sigmas[self.step_index_of(timestep)])
        return sample / ((sigma ** 2 + 1) ** 0.5)

    def add_noise(self, original_samples: torch.Tensor, noise: torch.Tensor, timesteps) -> torch.Tensor:
        idx = [self.step_index_of(t) for t in timesteps]
        sigma = self.sigmas[idx].flatten().to(original_samples.device, original_samples.dtype)
        while sigma.dim() < original_samples.dim():
            sigma = sigma.unsqueeze(-1)
        return original_samples + noise * sigma

    def _sigma_pair(self, timestep):
        i = self.step_index_of(timestep)
        return i, float(self.sigmas[i]), float(self.sigmas[i + 1])

    def _eps_and_original(self, model_output, sample, sigma: float):
        p = self.config["prediction_type"]
        return predicted_eps(p, model_output, sample, sigma), predicted_original(p, model_output, sample, sigma)


class EulerDiscreteScheduler(_SigmaScheduler):
    """Euler method on the probability-flow ODE dx/dsigma = eps (Karras et al. 2022, Algorithm 1 without churn):
    x' = x + (sigma' - sigma) eps."""

    def step(self, model_output: torch.Tensor, timestep, sample: torch.Tensor, **kw):
        _, sigma, sigma_next = self._sigma_pair(timestep)
        eps, original = self._eps_and_original(model_output, sample, sigma)
        return _StepOutput(sample + (sigma_next - sigma) * eps, original)


def ancestral_sigmas(sigma: float, sigma_next: float):
    """(sigma_down, sigma_up) of an ancestral step with eta = 1: sigma_up^2 = sigma'^2 (sigma^2 - sigma'^2) / sigma^2,
    sigma_down^2 = sigma'^2 - sigma_up^2."""
    sigma_up = (sigma_next ** 2 * (sigma ** 2 - sigma_next ** 2) / sigma ** 2) ** 0.5
    return (sigma_next ** 2 - sigma_up ** 2) ** 0.5, sigma_up


class EulerAncestralDiscreteScheduler(_SigmaScheduler):
    """Euler ancestral (k-diffusion `sample_euler_ancestral`, eta = 1, the diffusers-0.10 scheduler):
    x' = x + (sigma_down - sigma) eps + sigma_up z with z ~ N(0, I).  `step` takes z as `noise=` (or draws it from
    `generator`)."""

    def step(self, model_output: torch.Tensor, timestep, sample: torch.Tensor, noise: Optional[torch.Tensor] = None,
             generator: Optional[torch.Generator] = None, **kw):
        _, sigma, sigma_next = self._sigma_pair(timestep)
        sigma_down, sigma_up = ancestral_sigmas(sigma, sigma_next)
        if noise is None:
            noise = torch.randn(sample.shape, generator=generator, dtype=sample.dtype).to(sample.device)
        eps, original = self._eps_and_original(model_output, sample, sigma)
        prev = sample + (sigma_down - sigma) * eps + sigma_up * noise
        return _StepOutput(prev, original)


class DPMSolverMultistepScheduler(_SigmaScheduler):
    """DPM-Solver++(2M) in sigma space (Lu et al. 2022; k-diffusion `sample_dpmpp_2m`):
    D = x0 (x - sigma eps for an epsilon model), h = log sigma - log sigma',
      first order:  x' = (sigma'/sigma) x - expm1(-h) D
      second order: x' = (sigma'/sigma) x - expm1(-h) ((1 + 1/2r) D - (1/2r) D_prev),  r = h_prev / h.
    The first step of a run (or a step that does not follow the previous one) is first order, and the step to
    sigma' = 0 returns D."""
    order = 2

    def _reset(self):
        self._prev: Optional[tuple] = None     # (step index, D) of the last step

    def step(self, model_output: torch.Tensor, timestep, sample: torch.Tensor, **kw):
        i, sigma, sigma_next = self._sigma_pair(timestep)
        denoised = predicted_original(self.config["prediction_type"], model_output, sample, sigma)
        prev, self._prev = self._prev, (i, denoised)
        if sigma_next == 0:
            return _StepOutput(denoised, denoised)
        h = math.log(sigma) - math.log(sigma_next)
        e = math.expm1(-h)
        if prev is None or prev[0] != i - 1:
            return _StepOutput((sigma_next / sigma) * sample - e * denoised, denoised)
        r = (math.log(float(self.sigmas[i - 1])) - math.log(sigma)) / h
        d = (1 + 1 / (2 * r)) * denoised - (1 / (2 * r)) * prev[1]
        return _StepOutput((sigma_next / sigma) * sample - e * d, denoised)


SIGMA_SCHEDULERS = (LMSDiscreteScheduler, EulerDiscreteScheduler, EulerAncestralDiscreteScheduler,
                    DPMSolverMultistepScheduler)

# Columns of a step-form row (see `step_form`).
FORM_COLUMNS = ("alpha", "a", "b", "gamma", "slot", "row")


def history_length(scheduler) -> int:
    """Entries the step form keeps: 4 for LMS, 2 for DPM++ 2M, 1 for Euler (ancestral)."""
    if isinstance(scheduler, LMSDiscreteScheduler):
        return 4
    return 2 if isinstance(scheduler, DPMSolverMultistepScheduler) else 1


def step_form(scheduler, step_index: int, first: bool):
    """The step of `scheduler` at schedule position `step_index` as one linear update per image, in float64:
        q      = a x + b out                                        (the new history entry)
        x_next = alpha x + (beta0 q + beta1 h1 + beta2 h2 + beta3 h3) + gamma z
    with out the (guided) model output and h_k the entry k steps old.  `first`: no earlier step of this run (DPM++ 2M's
    first step is first order).  Returns (alpha, a, b, [beta0..beta3], gamma).  Any other scheduler class raises
    TypeError.
    For a v-prediction scheduler, eps = sigma/(sigma^2+1) x + v/sqrt(sigma^2+1) is linear in x and v, so its form is the
    epsilon form with a_v = a + b sigma/(sigma^2+1) and b_v = b/sqrt(sigma^2+1); alpha, beta and gamma are unchanged."""
    alpha, a, b, beta, gamma = _eps_step_form(scheduler, step_index, first)
    if scheduler.config["prediction_type"] == "epsilon":
        return alpha, a, b, beta, gamma
    sigma = float(scheduler.sigmas[step_index])
    return alpha, a + b * sigma / (sigma * sigma + 1.0), b / math.sqrt(sigma * sigma + 1.0), beta, gamma


def _eps_step_form(scheduler, step_index: int, first: bool):
    """`step_form` for an epsilon model: out = eps."""
    sch, i = scheduler, step_index
    if isinstance(sch, LMSDiscreteScheduler):
        # paint_with_words.py:506 -> order = min(step_index+1, 4) on the ABSOLUTE schedule index; missing history
        # (img2img starts mid-schedule) contributes nothing (a zeroed entry).
        coeffs = list(sch._coeffs[i]) if sch._coeffs is not None else sch._lms_coeffs(i, min(i + 1, 4))
        return 1.0, 0.0, 1.0, (coeffs + [0.0] * 4)[:4], 0.0
    if not isinstance(sch, _SigmaScheduler):
        raise TypeError(f"{type(sch).__name__} is not a supported scheduler; use one of "
                        + ", ".join(c.__name__ for c in SIGMA_SCHEDULERS))
    sigma, sigma_next = float(sch.sigmas[i]), float(sch.sigmas[i + 1])
    if isinstance(sch, EulerAncestralDiscreteScheduler):
        sigma_down, sigma_up = ancestral_sigmas(sigma, sigma_next)
        return 1.0, 0.0, 1.0, [sigma_down - sigma, 0.0, 0.0, 0.0], sigma_up
    if isinstance(sch, EulerDiscreteScheduler):
        return 1.0, 0.0, 1.0, [sigma_next - sigma, 0.0, 0.0, 0.0], 0.0
    # DPM++ 2M: q = D = x - sigma eps
    if sigma_next == 0:
        return 0.0, 1.0, -sigma, [1.0, 0.0, 0.0, 0.0], 0.0
    h = math.log(sigma) - math.log(sigma_next)
    e = math.expm1(-h)
    if first or i == 0:
        return sigma_next / sigma, 1.0, -sigma, [-e, 0.0, 0.0, 0.0], 0.0
    r = (math.log(float(sch.sigmas[i - 1])) - math.log(sigma)) / h
    return sigma_next / sigma, 1.0, -sigma, [-e * (1 + 1 / (2 * r)), e / (2 * r), 0.0, 0.0], 0.0
