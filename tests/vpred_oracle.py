"""Step-by-step restatements of the v-prediction branches of diffusers 0.30.2 ``DDIMScheduler`` (eta = 0),
``DPMSolverMultistepScheduler`` (DPM-Solver++(2M), midpoint, both ``final_sigmas_type`` endings) and ``PNDMScheduler``
(PLMS, skip_prk_steps), in x-space and in torch, written from diffusers' ``set_timesteps`` / ``step`` rather than from
the product's plan.  The alpha-bar table is fp32 like diffusers' (DPM-Solver++'s sigma table is derived from it in
float64); the arithmetic follows the dtype of the sample (the CPU tests feed float64, the GPU tests float32).  ``start``: image-to-image, a fresh scheduler (empty multistep state)
that begins at index ``start`` of the full timestep list.  Every ``step`` returns (prev_sample, x0 estimate)."""
import numpy as np
import torch

from oracle import restated as R


class _Base:
    def __init__(self, num_inference_steps, num_train_timesteps=1000, abar=None):
        self.n, self.n_train = num_inference_steps, num_train_timesteps
        self.abar = R.alphas_cumprod(n=num_train_timesteps) if abar is None else abar
        self.final_alpha_cumprod = self.abar[0]  # set_alpha_to_one=False

    def _abar(self, t, like):
        return (self.abar[t] if t >= 0 else self.final_alpha_cumprod).to(like.dtype)


class DDIM(_Base):
    def __init__(self, num_inference_steps, steps_offset=1, start=0, **kw):
        super().__init__(num_inference_steps, **kw)
        ratio = self.n_train // self.n
        ts = (np.arange(0, self.n) * ratio).round()[::-1].copy().astype(np.int64) + steps_offset
        self.timesteps = [int(t) for t in ts][start:]
        self.step_index = 0

    def step(self, model_output, sample):
        t = self.timesteps[self.step_index]
        prev_t = t - self.n_train // self.n
        alpha_prod_t = self._abar(t, sample)
        alpha_prod_t_prev = self._abar(prev_t, sample)
        beta_prod_t = 1 - alpha_prod_t
        pred_original_sample = alpha_prod_t ** 0.5 * sample - beta_prod_t ** 0.5 * model_output
        pred_epsilon = alpha_prod_t ** 0.5 * model_output + beta_prod_t ** 0.5 * sample
        pred_sample_direction = (1 - alpha_prod_t_prev) ** 0.5 * pred_epsilon
        prev = alpha_prod_t_prev ** 0.5 * pred_original_sample + pred_sample_direction
        self.step_index += 1
        return prev, pred_original_sample


class DPMSolverMultistep(_Base):
    def __init__(self, num_inference_steps, final_sigmas_type="zero", start=0, **kw):
        super().__init__(num_inference_steps, **kw)
        n, nt = self.n, self.n_train
        ts = np.linspace(0, nt - 1, n + 1).round()[::-1][:-1].copy().astype(np.int64)   # "linspace" spacing
        # diffusers evaluates this table in fp32 (1 - abar cancels near t = 0: sigma_min is off by ~7e-5 relative); it is
        # evaluated in float64 from the same fp32 abar here, like the product's plan, so that the comparison measures
        # the solver's algebra
        abar = self.abar.double()
        sigmas = (((1 - abar) / abar) ** 0.5).numpy()
        sigma_last = ((1 - abar[0]) / abar[0]) ** 0.5 if final_sigmas_type == "sigma_min" else 0.0
        sigmas = np.concatenate([np.interp(ts, np.arange(0, len(sigmas)), sigmas), [float(sigma_last)]])
        self.sigmas = torch.from_numpy(sigmas)
        self.all_timesteps = [int(t) for t in ts]
        self.timesteps = self.all_timesteps[start:]
        self.step_index = start
        self.model_outputs = [None, None]
        self.lower_order_nums = 0

    def _alpha_sigma_t(self, i, like):
        sigma = self.sigmas[i].to(like.dtype)
        alpha_t = 1 / ((sigma ** 2 + 1) ** 0.5)
        return alpha_t, sigma * alpha_t

    def step(self, model_output, sample):
        i, n = self.step_index, len(self.all_timesteps)
        lower_order_final = i == n - 1 and (n < 15 or self.sigmas[-1] == 0)
        lower_order_second = i == n - 2 and n < 15
        # convert_model_output, v branch
        alpha_s0, sigma_s0 = self._alpha_sigma_t(i, sample)
        x0 = alpha_s0 * sample - sigma_s0 * model_output
        self.model_outputs = [self.model_outputs[-1], x0]
        alpha_t, sigma_t = self._alpha_sigma_t(i + 1, sample)
        lambda_t = torch.log(alpha_t) - torch.log(sigma_t)
        lambda_s0 = torch.log(alpha_s0) - torch.log(sigma_s0)
        h = lambda_t - lambda_s0
        if self.lower_order_nums < 1 or lower_order_final or lower_order_second:
            prev = (sigma_t / sigma_s0) * sample - (alpha_t * (torch.exp(-h) - 1.0)) * x0
        else:
            alpha_s1, sigma_s1 = self._alpha_sigma_t(i - 1, sample)
            lambda_s1 = torch.log(alpha_s1) - torch.log(sigma_s1)
            m0, m1 = self.model_outputs[-1], self.model_outputs[-2]
            h_0 = lambda_s0 - lambda_s1
            r0 = h_0 / h
            D0, D1 = m0, (1.0 / r0) * (m0 - m1)
            prev = (sigma_t / sigma_s0) * sample - (alpha_t * (torch.exp(-h) - 1.0)) * D0 \
                - 0.5 * (alpha_t * (torch.exp(-h) - 1.0)) * D1
        if self.lower_order_nums < 2:
            self.lower_order_nums += 1
        self.step_index += 1
        return prev, x0


class PNDM(_Base):
    def __init__(self, num_inference_steps, steps_offset=1, start=0, **kw):
        super().__init__(num_inference_steps, **kw)
        ratio = self.n_train // self.n
        base = (np.arange(0, self.n) * ratio).round().astype(np.int64) + steps_offset
        plms = np.concatenate([base[:-1], base[-2:-1], base[-1:]])[::-1]
        self.timesteps = [int(t) for t in plms][start:]
        self.step_index = 0
        self.counter = 0
        self.ets = []
        self.cur_sample = None

    def _get_prev_sample(self, sample, timestep, prev_timestep, model_output):
        alpha_prod_t = self._abar(timestep, sample)
        alpha_prod_t_prev = self._abar(prev_timestep, sample)
        beta_prod_t = 1 - alpha_prod_t
        beta_prod_t_prev = 1 - alpha_prod_t_prev
        # v branch: the COMBINED output is converted, with this step's sample and timestep
        model_output = alpha_prod_t ** 0.5 * model_output + beta_prod_t ** 0.5 * sample
        sample_coeff = (alpha_prod_t_prev / alpha_prod_t) ** 0.5
        denom = alpha_prod_t * beta_prod_t_prev ** 0.5 + (alpha_prod_t * beta_prod_t * alpha_prod_t_prev) ** 0.5
        prev = sample_coeff * sample - (alpha_prod_t_prev - alpha_prod_t) * model_output / denom
        x0 = (sample - beta_prod_t ** 0.5 * model_output) / alpha_prod_t ** 0.5
        return prev, x0

    def step(self, model_output, sample):
        timestep = self.timesteps[self.step_index]
        prev_timestep = timestep - self.n_train // self.n
        if self.counter != 1:
            self.ets = self.ets[-3:]
            self.ets.append(model_output)
        else:
            prev_timestep = timestep
            timestep = timestep + self.n_train // self.n
        if len(self.ets) == 1 and self.counter == 0:
            self.cur_sample = sample
        elif len(self.ets) == 1 and self.counter == 1:
            model_output = (model_output + self.ets[-1]) / 2
            sample = self.cur_sample
            self.cur_sample = None
        elif len(self.ets) == 2:
            model_output = (3 * self.ets[-1] - self.ets[-2]) / 2
        elif len(self.ets) == 3:
            model_output = (23 * self.ets[-1] - 16 * self.ets[-2] + 5 * self.ets[-3]) / 12
        else:
            model_output = (55 * self.ets[-1] - 59 * self.ets[-2] + 37 * self.ets[-3] - 9 * self.ets[-4]) / 24
        self.counter += 1
        self.step_index += 1
        return self._get_prev_sample(sample, timestep, prev_timestep, model_output)


ORACLES = {"DDIM": DDIM, "DPMSolverMultistep": DPMSolverMultistep, "PNDM": PNDM}
