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
"""
from __future__ import annotations

from typing import List, Optional

import numpy as np
import torch
from scipy import integrate


class _StepOutput:
    def __init__(self, prev_sample, pred_original_sample):
        self.prev_sample = prev_sample
        self.pred_original_sample = pred_original_sample


class LMSDiscreteScheduler:
    order = 1

    def __init__(self, beta_start: float = 0.0001, beta_end: float = 0.02, beta_schedule: str = "linear",
                 num_train_timesteps: int = 1000):
        if beta_schedule == "linear":
            betas = np.linspace(beta_start, beta_end, num_train_timesteps, dtype=np.float32)
        elif beta_schedule == "scaled_linear":
            betas = np.linspace(beta_start ** 0.5, beta_end ** 0.5, num_train_timesteps, dtype=np.float32) ** 2
        else:
            raise NotImplementedError(beta_schedule)
        self.config = {"num_train_timesteps": num_train_timesteps, "beta_start": beta_start,
                       "beta_end": beta_end, "beta_schedule": beta_schedule}
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
        pred_original_sample = sample - sigma * model_output       # epsilon prediction
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
