"""Step-by-step restatements of diffusers 0.30.2 ``EulerDiscreteScheduler``, ``EulerAncestralDiscreteScheduler`` and
``LMSDiscreteScheduler`` (epsilon prediction, linear interpolation, no Karras sigmas), in x-space and in torch, written
from diffusers' ``set_timesteps`` / ``step`` rather than from the product's y-space plan.  The sigma table is fp32 like
diffusers'; the arithmetic follows the dtype of the sample (the CPU tests feed float64, the GPU tests float32).  The
LMS coefficients use ``scipy.integrate.quad(epsrel=1e-4)`` exactly as diffusers does."""
import numpy as np
import torch
from scipy import integrate

from oracle import restated as R


class _Sigmas:
    def __init__(self, num_inference_steps, timestep_spacing="linspace", steps_offset=1, num_train_timesteps=1000):
        n, nt = num_inference_steps, num_train_timesteps
        abar = R.alphas_cumprod(n=nt)
        if timestep_spacing == "linspace":
            ts = np.linspace(0, nt - 1, n, dtype=np.float32)[::-1].copy()
        elif timestep_spacing == "leading":
            step_ratio = nt // n
            ts = (np.arange(0, n) * step_ratio).round()[::-1].copy().astype(np.float32)
            ts += steps_offset
        elif timestep_spacing == "trailing":
            step_ratio = nt / n
            ts = (np.arange(nt, 0, -step_ratio)).round().copy().astype(np.float32)
            ts -= 1
        else:
            raise ValueError(timestep_spacing)
        sigmas = (((1 - abar) / abar) ** 0.5).numpy()
        sigmas = np.interp(ts, np.arange(0, len(sigmas)), sigmas)
        sigmas = np.concatenate([sigmas, [0.0]]).astype(np.float32)
        self.sigmas = torch.from_numpy(sigmas)
        self.timesteps = [float(t) for t in ts.astype(np.float32)]
        max_sigma = self.sigmas.max()
        if timestep_spacing in ("linspace", "trailing"):
            self.init_noise_sigma = float(max_sigma)
        else:
            self.init_noise_sigma = float((max_sigma ** 2 + 1) ** 0.5)
        self.step_index = 0

    def scale_model_input(self, sample, i):
        return sample / ((self.sigmas[i].to(sample.dtype) ** 2 + 1) ** 0.5)


class EulerDiscrete(_Sigmas):
    def step(self, eps, sample):
        """-> (prev_sample, pred_original_sample); s_churn = 0."""
        i = self.step_index
        sigma = self.sigmas[i].to(sample.dtype)
        x0 = sample - sigma * eps
        derivative = (sample - x0) / sigma
        dt = self.sigmas[i + 1].to(sample.dtype) - sigma
        self.step_index += 1
        return sample + derivative * dt, x0


class EulerAncestralDiscrete(_Sigmas):
    def step(self, eps, sample, noise):
        i = self.step_index
        sigma = self.sigmas[i].to(sample.dtype)
        x0 = sample - sigma * eps
        sigma_from, sigma_to = sigma, self.sigmas[i + 1].to(sample.dtype)
        sigma_up = (sigma_to ** 2 * (sigma_from ** 2 - sigma_to ** 2) / sigma_from ** 2) ** 0.5
        sigma_down = (sigma_to ** 2 - sigma_up ** 2) ** 0.5
        derivative = (sample - x0) / sigma
        dt = sigma_down - sigma
        prev = sample + derivative * dt
        self.step_index += 1
        return prev + noise * sigma_up, x0


class LMSDiscrete(_Sigmas):
    def __init__(self, *a, **kw):
        super().__init__(*a, **kw)
        self.derivatives = []

    def get_lms_coefficient(self, order, t, current_order):
        sig = self.sigmas.double()

        def lms_derivative(tau):
            prod = 1.0
            for k in range(order):
                if current_order == k:
                    continue
                prod *= (tau - float(sig[t - k])) / (float(sig[t - current_order]) - float(sig[t - k]))
            return prod

        return integrate.quad(lms_derivative, float(sig[t]), float(sig[t + 1]), epsrel=1e-4)[0]

    def step(self, eps, sample, order=4):
        i = self.step_index
        sigma = self.sigmas[i].to(sample.dtype)
        x0 = sample - sigma * eps
        self.derivatives.append((sample - x0) / sigma)
        if len(self.derivatives) > order:
            self.derivatives.pop(0)
        order = min(i + 1, order)
        coeffs = [self.get_lms_coefficient(order, i, o) for o in range(order)]
        prev = sample + sum(c * d for c, d in zip(coeffs, reversed(self.derivatives)))
        self.step_index += 1
        return prev, x0


ORACLES = {"EulerDiscrete": EulerDiscrete, "EulerAncestralDiscrete": EulerAncestralDiscrete,
           "LMSDiscrete": LMSDiscrete}


def oracle_step(sched, eps, sample, noise=None):
    """One step of any of the three, noise only for the ancestral one."""
    if isinstance(sched, EulerAncestralDiscrete):
        return sched.step(eps, sample, noise)
    return sched.step(eps, sample)
