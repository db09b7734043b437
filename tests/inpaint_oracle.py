"""Restatement of diffusers 0.30.2 ``StableDiffusionInpaintPipeline.__call__`` from mask processing to the final
latents, in float64 and x-space, written from diffusers rather than from the product's pipeline.  The UNet and the VAE
encoder are callables, and the scheduler steps are the restatements in ``sampler_oracle`` (Euler, Euler-ancestral,
LMS), ``vpred_oracle`` (v-prediction DDIM / DPM-Solver++ / PNDM) and ``oracle.restated`` (epsilon PNDM).  Epsilon
DDIM and DPM-Solver++ feed the v-prediction steps v = (eps - sigma_t x) / alpha_t: their updates only read x0 and
eps, which that v reproduces exactly.

What is restated:
* ``mask_processor`` (``VaeImageProcessor(do_binarize=True, do_convert_grayscale=True)``): binarise at 0.5 (0.5
  repaints); masked image = image * (mask < 0.5);
* ``get_timesteps``: t_start = n - min(int(n * strength), n), in float64, and ``set_begin_index(t_start)``;
* ``prepare_latents``: noise * init_noise_sigma at strength 1, else add_noise(image_latents, noise, timesteps[0]);
* ``prepare_mask_latents``: F.interpolate(mask, size=latent size) (nearest);
* the loop: UNet input cat([scale_model_input(latents)] * 2), for 9-channel UNets cat([that, mask, masked image
  latents], 1); guidance; ``scheduler.step``; for 4-channel UNets latents = (1 - m) init + m latents with init =
  add_noise(image_latents, noise, timesteps[i + 1]), or the image latents after the last step.
"""
import numpy as np
import torch
import torch.nn.functional as F

import sampler_oracle as SO
import vpred_oracle as V
from oracle import restated as R


def get_timesteps(num_inference_steps, strength):
    """-> t_start (diffusers' int() of a float64 product)."""
    init_timestep = min(int(num_inference_steps * strength), num_inference_steps)
    return max(num_inference_steps - init_timestep, 0)


def prepare_mask(image, mask):
    """-> (binarised mask (B, 1, H, W), masked image); ``mask`` (B | 1, 1, H, W) or (H, W)."""
    image = torch.as_tensor(image).double()
    mask = torch.as_tensor(mask).double().clone()
    if mask.dim() == 2:
        mask = mask[None, None]
    mask[mask < 0.5] = 0
    mask[mask >= 0.5] = 1
    mask = mask.expand(image.shape[0], 1, *image.shape[2:])
    return mask, image * (mask < 0.5)


class _DDIM(V.DDIM):
    def __init__(self, n, prediction_type, start=0, **kw):
        super().__init__(n, start=start, **kw)
        self.eps = prediction_type == "epsilon"
        self.init_noise_sigma = 1.0

    def step(self, out, sample, noise=None):
        if self.eps:
            a = self._abar(self.timesteps[self.step_index], sample)
            out = (out - (1 - a) ** 0.5 * sample) / a ** 0.5
        return super().step(out, sample)[0]

    def add_noise(self, x0, z, k):
        a = self._abar(self.timesteps[k], x0)
        return a ** 0.5 * x0 + (1 - a) ** 0.5 * z

    def scale(self, sample, i):
        return sample


class _DPM(V.DPMSolverMultistep):
    def __init__(self, n, prediction_type, start=0, **kw):
        super().__init__(n, start=start, **kw)
        self.eps, self.start = prediction_type == "epsilon", start
        self.init_noise_sigma = 1.0

    def step(self, out, sample, noise=None):
        if self.eps:
            alpha, sigma = self._alpha_sigma_t(self.step_index, sample)
            out = (out - sigma * sample) / alpha
        return super().step(out, sample)[0]

    def add_noise(self, x0, z, k):
        """With a begin index the sigma table is read at the step index (begin + k), not by timestep value."""
        alpha, sigma = self._alpha_sigma_t(self.start + k, x0)
        return alpha * x0 + sigma * z

    def scale(self, sample, i):
        return sample


class _PNDM:
    def __init__(self, n, prediction_type, start=0):
        assert start == 0
        self.abar = R.alphas_cumprod()
        self.eps = prediction_type == "epsilon"
        self.s = R.PNDM(n, abar=self.abar.double()) if self.eps else V.PNDM(n)
        self.timesteps = list(self.s.timesteps)
        self.i = 0
        self.init_noise_sigma = 1.0

    def step(self, out, sample, noise=None):
        t = self.timesteps[self.i]
        self.i += 1
        return self.s.step(out, t, sample) if self.eps else self.s.step(out, sample)[0]

    def add_noise(self, x0, z, k):
        a = self.abar[self.timesteps[k]].double()
        return a ** 0.5 * x0 + (1 - a) ** 0.5 * z

    def scale(self, sample, i):
        return sample


class _Sigma:
    def __init__(self, name, n, prediction_type="epsilon", start=0, **kw):
        assert start == 0 and prediction_type == "epsilon"
        self.s = SO.ORACLES[name](n, **kw)
        self.timesteps = self.s.timesteps
        self.init_noise_sigma = self.s.init_noise_sigma

    def step(self, out, sample, noise=None):
        return SO.oracle_step(self.s, out, sample, noise)[0]

    def add_noise(self, x0, z, k):
        return x0 + self.s.sigmas[k].double() * z

    def scale(self, sample, i):
        return self.s.scale_model_input(sample, i)


def make_scheduler(name, n, prediction_type="epsilon", start=0, **kw):
    """A fresh scheduler after ``set_timesteps(n)`` and ``set_begin_index(start)``: ``timesteps`` (from ``start``),
    ``step(model_output, sample[, noise]) -> prev``, ``add_noise(x0, z, k)`` at ``timesteps[k]``, ``scale`` (the
    ``scale_model_input`` of step i) and ``init_noise_sigma``."""
    if name == "DDIM":
        return _DDIM(n, prediction_type, start, **kw)
    if name == "DPMSolverMultistep":
        return _DPM(n, prediction_type, start, **kw)
    if name == "PNDM":
        return _PNDM(n, prediction_type, start)
    return _Sigma(name, n, prediction_type, start, **kw)


def inpaint(unet, encode, image, mask_image, noise, name, num_inference_steps, guidance_scale, strength=1.0,
            in_channels=4, prediction_type="epsilon", step_noise=None, model_outputs=None, record=None, **sched_kw):
    """-> final latents (B, c, h, w) float64.  ``unet(sample (2B, in_channels, h, w), t) -> (2B, c, h, w)``;
    ``encode(image (B, 3, H, W)) -> latents``, called for the full image (4-channel UNet or strength < 1), then for the
    masked image (9-channel UNet); ``noise``: the initial noise (B, c, h, w); ``step_noise(i)``: the ancestral noise
    of step i.  ``model_outputs``: per-step UNet outputs to use instead of calling ``unet`` (to check the scheduler
    and blend arithmetic alone); ``record`` receives the latents after every step."""
    mask, masked_image = prepare_mask(image, mask_image)
    start = get_timesteps(num_inference_steps, strength)
    sched = make_scheduler(name, num_inference_steps, prediction_type, start, **sched_kw)
    noise = torch.as_tensor(noise).double()
    is_strength_max = strength == 1.0
    image_latents = masked_image_latents = None
    if in_channels == 4 or not is_strength_max:
        image_latents = torch.as_tensor(encode(torch.as_tensor(image))).double()
    if in_channels == 9:
        masked_image_latents = torch.as_tensor(encode(masked_image)).double()
    latents = noise * sched.init_noise_sigma if is_strength_max else sched.add_noise(image_latents, noise, 0)
    m = F.interpolate(mask, size=tuple(latents.shape[2:]))
    b = latents.shape[0]
    n = len(sched.timesteps)
    for i, t in enumerate(sched.timesteps):
        x_in = sched.scale(torch.cat([latents] * 2), i)
        if in_channels == 9:
            x_in = torch.cat([x_in, torch.cat([m] * 2), torch.cat([masked_image_latents] * 2)], dim=1)
        out = unet(x_in, t) if model_outputs is None else model_outputs[i]
        out = torch.as_tensor(out).double()
        eps = R.cfg_combine(out[:b], out[b:], guidance_scale)
        latents = sched.step(eps, latents, None if step_noise is None else torch.as_tensor(step_noise(i)).double())
        if in_channels == 4:
            init = image_latents
            if i < n - 1:
                init = sched.add_noise(image_latents, noise, i + 1)
            latents = (1 - m) * init + m * latents
        if record is not None:
            record.append(latents.clone())
    return latents
