"""Host side of the fused CFG + scheduler-step kernel: per-step fp32 coefficients.

The reference does this math on the host, per element, in fp32: Python defers to diffusers
(``pipeline.py:475-476,504-505,565-569``), the in-tree spec is the Swift twin
(``swift/StableDiffusion/pipeline/Scheduler.swift:137-344`` PNDM/PLMS,
``DPMSolverMultistepScheduler.swift:27-245`` DPM-Solver++ 2M; DDIM == its first-order update,
``:153-174``).  Every one of those updates is *linear* in (x_t, eps, history), so here each
scheduler only produces, per step, the scalars of

    x_prev = cx * x + ce * eps + sum_i ch[i]    * hist[i]
    x0     = x0_cx * x + x0_ce * eps + sum_i x0_ch[i] * hist[i]

plus which history slots to overwrite; ``b200sd_cfg_scheduler_step`` applies them on the device
(one launch, also does classifier-free guidance and writes the next UNet input), so the denoising
loop never synchronises with the host.  Coefficients are computed in float64 and rounded once.

DDIM, DPM-Solver++ and PNDM also run v-prediction models (SD 2.0 / 2.1 768-v, ``prediction_type="v_prediction"``):
diffusers 0.30.2 converts the model output v to x0 = alpha_t x - sigma_t v or eps = alpha_t v + sigma_t x inside
``step``, which keeps every update linear in (x, v, history), so only the coefficients change.
"""
from __future__ import annotations

import dataclasses
import math
from typing import List

import numpy as np


@dataclasses.dataclass
class StepPlan:
    """One denoising step: UNet timestep + the linear-update coefficients."""
    timestep: int
    cx: float
    ce: float
    ch: List[float]
    x0_cx: float
    x0_ce: float
    x0_ch: List[float]
    n_hist: int = 0
    push_eps_slot: int = -1
    push_x0_slot: int = -1
    push_x_slot: int = -1
    # ancestral samplers: x_prev += noise_scale * z, z the Philox normals of the step's noise draw number
    # `noise_offset` (b200sd_cfg_scheduler_step_noised); -1: no noise this step
    noise_scale: float = 0.0
    noise_offset: int = -1


def alphas_cumprod(beta_start=0.00085, beta_end=0.012, n=1000, schedule="scaled_linear"):
    """fp32 like the reference (Scheduler.swift:168-186)."""
    if schedule == "scaled_linear":
        betas = np.linspace(np.float32(beta_start) ** 0.5, np.float32(beta_end) ** 0.5, n, dtype=np.float32) ** 2
    elif schedule == "linear":
        betas = np.linspace(beta_start, beta_end, n, dtype=np.float32)
    else:
        raise ValueError(f"unknown beta schedule {schedule}")
    return np.cumprod((1.0 - betas).astype(np.float32), dtype=np.float32)


def alphas_cumprod_diffusers(beta_start=0.00085, beta_end=0.012, n=1000, schedule="scaled_linear"):
    """The fp32 table of diffusers 0.30.2 (torch.linspace + torch.cumprod), which differs from ``alphas_cumprod`` in
    the last bits (sigma_max by 1.5e-6 relative): the Euler / LMS samplers restate diffusers, so they use this one."""
    import torch
    if schedule == "scaled_linear":
        betas = torch.linspace(beta_start ** 0.5, beta_end ** 0.5, n, dtype=torch.float32) ** 2
    elif schedule == "linear":
        betas = torch.linspace(beta_start, beta_end, n, dtype=torch.float32)
    else:
        raise ValueError(f"unknown beta schedule {schedule}")
    return torch.cumprod(1.0 - betas, dim=0).numpy()


class _Base:
    init_noise_sigma = 1.0
    n_hist_slots = 4

    def __init__(self, num_inference_steps, num_train_timesteps=1000, beta_start=0.00085, beta_end=0.012,
                 beta_schedule="scaled_linear"):
        if num_inference_steps < 1:
            raise ValueError("num_inference_steps must be >= 1")
        self.n = int(num_inference_steps)
        self.n_train = int(num_train_timesteps)
        self.abar = alphas_cumprod(beta_start, beta_end, num_train_timesteps, beta_schedule).astype(np.float64)
        self._beta_args = (beta_start, beta_end, num_train_timesteps, beta_schedule)

    def scale_model_input(self, x, t):  # identity for DDIM / PNDM / DPM (pipeline.py:504)
        return x

    def input_scale(self, i: int) -> float:
        """x = input_scale(i) * (loop state) before step i; i == len(plan) is the end of the loop.  1 for the
        schedulers whose loop state is the latent itself."""
        return 1.0

    @property
    def timesteps(self):
        return [p.timestep for p in self.plan()]

    def plan(self, start: int = 0) -> List[StepPlan]:
        """Steps ``start`` .. end of the schedule, with the multistep state starting empty at ``start`` (what a
        fresh Swift scheduler does when the pipeline feeds it ``calculateTimesteps(strength)``)."""
        raise NotImplementedError

    # ---- image-to-image (Scheduler.swift:83-114) ----
    def start_step(self, strength: float) -> int:
        """max(inferenceStepCount - Int(Float(inferenceStepCount) * strength), 0)."""
        return max(self.n - int(np.float32(self.n) * np.float32(strength)), 0)

    def calculate_timesteps(self, strength=None):
        ts = self.timesteps
        return ts if strength is None else ts[self.start_step(strength):]

    def add_noise(self, original_sample, noise, strength):
        """sqrt(abar_t) * x0 + sqrt(1 - abar_t) * noise at t = timeSteps[startStep]."""
        t = self.timesteps[self.start_step(strength)]
        a = np.float32(self.abar[t])
        return np.float32(np.sqrt(a)) * original_sample + np.float32(np.sqrt(np.float32(1.0) - a)) * noise

    # ---- inpainting (diffusers 0.30.2 StableDiffusionInpaintPipeline) ----
    def inpaint_start_step(self, strength: float) -> int:
        """``get_timesteps``: n - min(int(n * strength), n) in float64 (the image-to-image rule, ``start_step``, rounds
        in float32 and can differ by one, e.g. n = 100, strength = 0.29)."""
        return max(self.n - min(int(self.n * float(strength)), self.n), 0)

    def noise_coeffs(self, j: int):
        """(a, b) of diffusers' ``add_noise(x0, z, timesteps[j])`` = a x0 + b z, in the loop's state space; ``j``
        indexes the full plan (PNDM's repeated timestep is an entry of its own).  DDIM / PNDM: sqrt(abar_t),
        sqrt(1 - abar_t) from diffusers' fp32 alpha-bar table."""
        t = self.plan()[j].timestep
        a = float(alphas_cumprod_diffusers(*self._beta_args)[t])
        return math.sqrt(a), math.sqrt(1.0 - a)

    def blend_coeffs(self, start: int = 0):
        """Per step of ``plan(start)``: the (a, b) of the inpainting blend after that step, x' = m x' + (1 - m)(a x0_img +
        b z): ``add_noise`` at the next timestep (``timesteps[k + 1]``, what the inpaint pipeline calls after step k),
        and on the last step (1 / s_N, 0) -- the image latents themselves, divided by the final input scale."""
        n_plan = len(self.plan(start))
        out = [self.noise_coeffs(start + k + 1) for k in range(n_plan - 1)]
        out.append((1.0 / self.input_scale(start + n_plan), 0.0))
        return out


PREDICTION_TYPES = ("epsilon", "v_prediction")
#: the scheduler classes that take ``prediction_type``
PREDICTION_TYPE_SCHEDULERS = ("DDIM", "DPMSolverMultistep", "PNDM")


def check_prediction_type(value):
    if value not in PREDICTION_TYPES:
        raise ValueError(f"prediction_type must be one of {PREDICTION_TYPES}, got {value!r}")
    return value


class DDIMScheduler(_Base):
    """eta = 0, 'leading' spacing, steps_offset 1, set_alpha_to_one False.  ``prediction_type="v_prediction"``:
    x0 = alpha_t x - sigma_t v and eps = sigma_t x + alpha_t v (diffusers 0.30.2 ``DDIMScheduler.step``)."""

    def __init__(self, num_inference_steps, steps_offset=1, prediction_type="epsilon", **kw):
        super().__init__(num_inference_steps, **kw)
        self.steps_offset = steps_offset
        self.prediction_type = check_prediction_type(prediction_type)

    def plan(self, start=0):
        ratio = self.n_train // self.n
        ts = [int(round(i * ratio)) + self.steps_offset for i in range(self.n)][::-1]
        out = []
        for t in ts[start:]:
            tp = t - ratio
            a_t = self.abar[t]
            a_p = self.abar[tp] if tp >= 0 else self.abar[0]
            if self.prediction_type == "epsilon":
                x0_cx = 1.0 / math.sqrt(a_t)
                x0_ce = -math.sqrt(1 - a_t) / math.sqrt(a_t)
                cx = math.sqrt(a_p) * x0_cx
                ce = math.sqrt(a_p) * x0_ce + math.sqrt(1 - a_p)
            else:  # x' = alpha_p x0 + sigma_p eps
                al_t, sg_t, al_p, sg_p = math.sqrt(a_t), math.sqrt(1 - a_t), math.sqrt(a_p), math.sqrt(1 - a_p)
                x0_cx, x0_ce = al_t, -sg_t
                cx = al_p * al_t + sg_p * sg_t
                ce = sg_p * al_t - al_p * sg_t
            out.append(StepPlan(t, cx, ce, [0.0] * 4, x0_cx, x0_ce, [0.0] * 4))
        return out


class DPMSolverMultistepScheduler(_Base):
    """DPM-Solver++(2M) midpoint, 'linspace' spacing; first step and (for < 15
    steps) the last two steps are first order (DPMSolverMultistepScheduler.swift:216-244).
    History ring: x0 of the previous step in slots 0/1.  The solver works on x0 estimates, so
    ``prediction_type="v_prediction"`` only changes how x0 is read from the model output: x0 = alpha_t x - sigma_t v
    (diffusers 0.30.2 ``convert_model_output``).

    ``final_sigmas_type``: how the LAST step ends.  ``"sigma_min"``: at the first training timestep's (alpha, sigma),
    what the in-tree Swift scheduler does (``alpha_t[0] / sigma_t[0]``, DPMSolverMultistepScheduler.swift:214-222).
    ``"zero"``: diffusers 0.30.2's default, which the reference's PYTHON pipeline runs (pipeline.py:565-569 ->
    ``scheduler.step``): the final sigma is 0, the last step is always first order and lands exactly on the
    denoised estimate x0."""

    def __init__(self, num_inference_steps, final_sigmas_type="sigma_min", prediction_type="epsilon", **kw):
        super().__init__(num_inference_steps, **kw)
        if final_sigmas_type not in ("sigma_min", "zero"):
            raise ValueError(f"final_sigmas_type must be 'sigma_min' or 'zero', got {final_sigmas_type!r}")
        self.final_sigmas_type = final_sigmas_type
        self.prediction_type = check_prediction_type(prediction_type)

    def plan(self, start=0):
        n = self.n
        ts = [int(round(v)) for v in np.linspace(0, self.n_train - 1, n + 1)[1:][::-1]]
        alpha = np.sqrt(self.abar)
        sigma = np.sqrt(1.0 - self.abar)
        lam = np.log(alpha) - np.log(sigma)
        out = []
        lower_order_stepped = 0
        for i, t in enumerate(ts):
            if i < start:
                continue
            p = ts[i + 1] if i + 1 < n else 0
            lower_final = (i == n - 1) and n < 15
            lower_second = (i == n - 2) and n < 15
            first = lower_order_stepped < 1 or lower_final or lower_second
            if self.prediction_type == "epsilon":
                x0_cx = 1.0 / alpha[t]
                x0_ce = -sigma[t] / alpha[t]
            else:
                x0_cx, x0_ce = alpha[t], -sigma[t]
            h = lam[p] - lam[t]
            A = -alpha[p] * (math.exp(-h) - 1.0)
            ch = [0.0] * 4
            slot, prev_slot = i % 2, (i - 1) % 2
            if i == n - 1 and self.final_sigmas_type == "zero":
                cx, ce, n_hist = x0_cx, x0_ce, 0      # sigma_next = 0, alpha_next = 1: x_prev = x0 (first order)
            elif first:
                cx = sigma[p] / sigma[t] + A * x0_cx
                ce = A * x0_ce
                n_hist = 0
            else:
                h0 = lam[t] - lam[ts[i - 1]]
                r0 = h0 / h
                c0 = A * (1.0 + 0.5 / r0)
                cx = sigma[p] / sigma[t] + c0 * x0_cx
                ce = c0 * x0_ce
                ch[prev_slot] = -0.5 * A / r0
                n_hist = 2
            out.append(StepPlan(t, cx, ce, ch, x0_cx, x0_ce, [0.0] * 4, n_hist=n_hist, push_x0_slot=slot))
            if lower_order_stepped < 2:
                lower_order_stepped += 1
        return out

    def noise_coeffs(self, j):
        """diffusers' ``add_noise`` with a begin index set (the inpaint pipeline always sets one) reads the sigma table
        at the STEP index j, not by timestep value: alpha_t = 1 / sqrt(sigma_j^2 + 1), sigma_t = sigma_j alpha_t, sigma_j
        evaluated in float64 from diffusers' fp32 alpha-bar table."""
        t = self.plan()[j].timestep
        a = float(alphas_cumprod_diffusers(*self._beta_args)[t])
        sig = math.sqrt((1.0 - a) / a)
        alpha_t = 1.0 / math.sqrt(sig * sig + 1.0)
        return alpha_t, sig * alpha_t


class PNDMScheduler(_Base):
    """PLMS (skip_prk_steps) (Scheduler.swift:137-344): num_steps + 1 UNet calls
    (the second timestep is visited twice).  History ring: eps in slots 0..2, the saved first
    sample (`currentSample`) in slot 3.

    ``prediction_type="v_prediction"`` (diffusers 0.30.2 ``_get_prev_sample``): the ring keeps the RAW model outputs v,
    and only their Adams-Bashforth combination e is converted, with the step's sample s and (shifted) timestep t:
    eps = alpha_t e + sigma_t s.  Converting each v before combining would give another sampler after the first step."""

    def __init__(self, num_inference_steps, steps_offset=1, prediction_type="epsilon", **kw):
        super().__init__(num_inference_steps, **kw)
        self.steps_offset = steps_offset
        self.prediction_type = check_prediction_type(prediction_type)

    def _prev_coeffs(self, t, tp):
        a_t = self.abar[t]
        a_p = self.abar[max(0, tp)]
        b_t, b_p = 1 - a_t, 1 - a_p
        sample_coeff = math.sqrt(a_p / a_t)
        denom = a_t * math.sqrt(b_p) + math.sqrt(a_t * b_t * a_p)
        return sample_coeff, -(a_p - a_t) / denom

    def plan(self, start=0):
        ratio = self.n_train // self.n
        fwd = [int(round(i * float(ratio))) + self.steps_offset for i in range(self.n)]
        ts = fwd[:-1]
        ts = ts + [ts[-1]] if ts else []
        ts = (ts + [fwd[-1]])[::-1]
        # image-to-image: the Swift pipeline slices this list (timeSteps[startStep...], Scheduler.swift:109-114) and
        # feeds it to a fresh scheduler, whose counter-driven branches then apply to whatever comes first
        ts = ts[start:]
        alpha = np.sqrt(self.abar)
        sigma = np.sqrt(1.0 - self.abar)
        out = []
        n_ets = 0  # eps pushed so far
        for counter, t_unet in enumerate(ts):
            t, tp = t_unet, t_unet - ratio
            ch = [0.0] * 4
            x0_ch = [0.0] * 4
            push_eps, push_x = -1, -1
            if counter != 1:
                push_eps = n_ets % 3
                n_ets += 1
                k = min(n_ets, 4)  # entries of `ets` available including the current eps
            else:
                tp, t = t, t + ratio
                k = 0
            sc, mc = self._prev_coeffs(t, tp)
            slot_back = lambda b: (n_ets - b) % 3  # ets[back: b], b >= 2 (b == 1 is the current eps)
            if counter == 0:
                w_cur, w_hist, use_saved = 1.0, {}, False
                push_x = 3
            elif counter == 1:
                w_cur, w_hist, use_saved = 0.5, {(n_ets - 1) % 3: 0.5}, True
            elif k == 2:
                w_cur, w_hist, use_saved = 1.5, {slot_back(2): -0.5}, False
            elif k == 3:
                w_cur, w_hist, use_saved = 23 / 12, {slot_back(2): -16 / 12, slot_back(3): 5 / 12}, False
            else:
                w_cur = 55 / 24
                w_hist = {slot_back(2): -59 / 24, slot_back(3): 37 / 24, slot_back(4): -9 / 24}
                use_saved = False
            # x_prev = sc * sample + mc * eps' ; x0 = (sample - sigma_t eps') / alpha_t ; e = w_cur out + sum w h ;
            # eps' = e (epsilon) or alpha_t e + sigma_t sample (v): x_prev = s_x sample + s_e e, x0 = x0_x sample + x0_e e
            a_t, s_t = alpha[t], sigma[t]
            if self.prediction_type == "epsilon":
                s_x, s_e, x0_x, x0_e = sc, mc, 1.0 / a_t, -s_t / a_t
            else:
                s_x, s_e, x0_x, x0_e = sc + mc * s_t, mc * a_t, a_t, -s_t
            cx = 0.0 if use_saved else s_x
            x0_cx = 0.0 if use_saved else x0_x
            if use_saved:
                ch[3] += s_x
                x0_ch[3] += x0_x
            ce = s_e * w_cur
            x0_ce = x0_e * w_cur
            for s, wv in w_hist.items():
                ch[s] += s_e * wv
                x0_ch[s] += x0_e * wv
            n_hist = 4 if (use_saved or w_hist) else 0
            out.append(StepPlan(t_unet, cx, ce, ch, x0_cx, x0_ce, x0_ch, n_hist=n_hist, push_eps_slot=push_eps,
                                push_x_slot=push_x))
        return out


class _SigmaScheduler(_Base):
    """Shared part of diffusers 0.30.2 ``EulerDiscreteScheduler``, ``EulerAncestralDiscreteScheduler`` and
    ``LMSDiscreteScheduler`` (the classes the reference imports, pipeline.py:11-18), epsilon prediction, linear
    interpolation, no Karras sigmas.  Defaults are ``X.from_config(<SD 1.x / 2.1-base scheduler config>)``, what the
    reference CLI runs for ``--scheduler X``: scaled_linear betas, steps_offset 1, ``timestep_spacing="linspace"``.

    These samplers work on x = x0 + sigma * noise.  The device loop keeps y = x / s, s = sqrt(sigma^2 + 1), instead:
    y is exactly what ``scale_model_input`` hands the UNet, and every update stays linear in (y, eps, history), so
    the plan is the same StepPlan the other schedulers produce.  The final sigma is 0, so the last y is x."""
    SPACINGS = ("linspace", "leading", "trailing")

    def __init__(self, num_inference_steps, timestep_spacing="linspace", steps_offset=1, num_train_timesteps=1000,
                 beta_start=0.00085, beta_end=0.012, beta_schedule="scaled_linear"):
        super().__init__(num_inference_steps, num_train_timesteps, beta_start, beta_end, beta_schedule)
        if timestep_spacing not in self.SPACINGS:
            raise ValueError(f"timestep_spacing must be one of {self.SPACINGS}, got {timestep_spacing!r}")
        self.timestep_spacing, self.steps_offset = timestep_spacing, int(steps_offset)
        n, nt = self.n, self.n_train
        if timestep_spacing == "linspace":
            ts = np.linspace(0, nt - 1, n, dtype=np.float32)[::-1].copy()
        elif timestep_spacing == "leading":
            ts = (np.arange(0, n) * (nt // n)).round()[::-1].copy().astype(np.float32)
            ts += self.steps_offset
        else:
            ts = np.arange(nt, 0, -nt / n).round().copy().astype(np.float32)
            ts -= 1
        abar = alphas_cumprod_diffusers(beta_start, beta_end, num_train_timesteps, beta_schedule)
        table = ((1 - abar) / abar) ** 0.5
        #: the (possibly fractional) timesteps at which sigma is interpolated
        self.sigma_timesteps = [float(t) for t in ts]
        #: fp32 sigmas of the steps, then the final 0
        self.sigmas = np.concatenate([np.interp(ts, np.arange(0, len(table)), table), [0.0]]).astype(np.float32)
        smax = self.sigmas.max()
        self.init_noise_sigma = float(smax if timestep_spacing != "leading" else (smax * smax + np.float32(1)) ** 0.5)

    def input_scale(self, i):
        return math.sqrt(float(self.sigmas[i]) ** 2 + 1.0)

    def plan(self, start=0):
        if start:
            raise ValueError(f"{type(self).__name__} has no image-to-image schedule")
        out = []
        for i, t in enumerate(self.sigma_timesteps):
            sig, sig_next = float(self.sigmas[i]), float(self.sigmas[i + 1])
            s, s_next = self.input_scale(i), self.input_scale(i + 1)
            # the reference feeds the UNet np.array([t, t], np.float16) (pipeline.py:511-514)
            st = StepPlan(float(np.float16(t)), s / s_next, 0.0, [0.0] * 4, s, -sig, [0.0] * 4)
            self._update(st, i, sig, sig_next, s_next)
            out.append(st)
        return out

    def _update(self, st, i, sig, sig_next, s_next):
        """Fill ce / ch / history / noise of step i (cx = s / s', x0 = s y - sigma eps are common)."""
        raise NotImplementedError

    def noise_coeffs(self, j):
        """``add_noise`` = x0 + sigma_j z (sigma table at step index j), divided by s_j = sqrt(sigma_j^2 + 1): the loop
        state is y = x / s."""
        sig, s = float(self.sigmas[j]), self.input_scale(j)
        return 1.0 / s, sig / s


class EulerDiscreteScheduler(_SigmaScheduler):
    """x' = x + (sigma' - sigma) eps (s_churn = 0: no noise)."""

    def _update(self, st, i, sig, sig_next, s_next):
        st.ce = (sig_next - sig) / s_next


class EulerAncestralDiscreteScheduler(_SigmaScheduler):
    """The Euler step to sigma_down, then + sigma_up z.  Step i draws its z as noise draw number i."""

    @staticmethod
    def sigma_up_down(sig, sig_next):
        up = math.sqrt(sig_next ** 2 * (sig ** 2 - sig_next ** 2) / sig ** 2)
        return up, math.sqrt(sig_next ** 2 - up ** 2)

    def _update(self, st, i, sig, sig_next, s_next):
        up, down = self.sigma_up_down(sig, sig_next)
        st.ce = (down - sig) / s_next
        if up > 0.0:
            st.noise_scale, st.noise_offset = up / s_next, i


class LMSDiscreteScheduler(_SigmaScheduler):
    """Linear multistep of order min(step + 1, 4): x' = x + sum_k c_k eps_{i-k}, c_k the integral from sigma_i to
    sigma_{i+1} of the k-th Lagrange basis polynomial over the nodes sigma_i .. sigma_{i-order+1}.  diffusers integrates
    with ``scipy.integrate.quad``; these cubics are integrated exactly here.  History ring: eps of step i in slot i % 3
    (the three previous eps are all an order-4 step reads)."""
    order = 4

    def lms_coefficients(self, i):
        order = min(i + 1, self.order)
        nodes = [float(self.sigmas[i - m]) for m in range(order)]
        a, b = float(self.sigmas[i]), float(self.sigmas[i + 1])
        P = np.polynomial.polynomial
        out = []
        for k in range(order):
            poly = np.array([1.0])
            for m in range(order):
                if m != k:
                    poly = P.polymul(poly, np.array([-nodes[m], 1.0]) / (nodes[k] - nodes[m]))
            prim = P.polyint(poly)
            out.append(float(P.polyval(b, prim) - P.polyval(a, prim)))
        return out

    def _update(self, st, i, sig, sig_next, s_next):
        c = self.lms_coefficients(i)
        st.ce = c[0] / s_next
        for k in range(1, len(c)):
            st.ch[(i - k) % 3] = c[k] / s_next
        st.n_hist = 3 if len(c) > 1 else 0
        st.push_eps_slot = i % 3


class LCMScheduler(_Base):
    """diffusers 0.30.2 ``LCMScheduler`` (latent consistency models), restated from its ``set_timesteps`` and ``step``.

    Timesteps: with k = n_train // original_inference_steps, origin = (arange(1, original_inference_steps + 1) k - 1)
    reversed, the n steps are origin[floor(linspace(0, len(origin), n, endpoint=False))] (4 of 50: 999, 759, 499, 259).
    Step i at t, prev = timesteps[i + 1] (t itself on the last step), abar from diffusers' fp32 table:
        s = timestep_scaling t,  c_skip = 0.25 / (s^2 + 0.25),  c_out = s / sqrt(s^2 + 0.25)      (sigma_data = 0.5)
        x0 = (x - sqrt(1 - abar_t) eps) / sqrt(abar_t)    (v_prediction: x0 = sqrt(abar_t) x - sqrt(1 - abar_t) v)
        denoised = c_out x0 + c_skip x
        x' = sqrt(abar_prev) denoised + sqrt(1 - abar_prev) z   on every step but the last, where x' = denoised.
    All of it is linear in (x, eps, z): the plan's x0 terms are ``denoised``, the noise is noise draw number i with
    noise_scale sqrt(1 - abar_prev).  z is the in-kernel Philox stream keyed by the seed (as for Euler-ancestral), so
    the images are not bit-compatible with diffusers' torch-generator noise.  No image-to-image schedule: LCM's
    ``strength`` changes the timesteps themselves."""

    def __init__(self, num_inference_steps, original_inference_steps=50, timestep_scaling=10.0,
                 prediction_type="epsilon", num_train_timesteps=1000, beta_start=0.00085, beta_end=0.012,
                 beta_schedule="scaled_linear"):
        super().__init__(num_inference_steps, num_train_timesteps, beta_start, beta_end, beta_schedule)
        self.original_inference_steps = int(original_inference_steps)
        if self.n > self.original_inference_steps:
            raise ValueError(f"num_inference_steps={self.n} exceeds the LCM schedule's original_inference_steps="
                             f"{self.original_inference_steps}")
        self.timestep_scaling = float(timestep_scaling)
        self.prediction_type = check_prediction_type(prediction_type)
        self.abar = alphas_cumprod_diffusers(beta_start, beta_end, num_train_timesteps, beta_schedule).astype(np.float64)
        k = self.n_train // self.original_inference_steps
        origin = (np.arange(1, self.original_inference_steps + 1) * k - 1)[::-1]
        idx = np.floor(np.linspace(0, len(origin), self.n, endpoint=False)).astype(np.int64)
        self.lcm_timesteps = [int(t) for t in origin[idx]]

    def plan(self, start=0):
        if start:
            raise ValueError("LCMScheduler has no image-to-image schedule")
        ts = self.lcm_timesteps
        out = []
        for i, t in enumerate(ts):
            last = i == len(ts) - 1
            a_t = self.abar[t]
            a_p = self.abar[t if last else ts[i + 1]]
            s = t * self.timestep_scaling
            c_skip = 0.25 / (s * s + 0.25)
            c_out = s / math.sqrt(s * s + 0.25)
            if self.prediction_type == "epsilon":
                x0_x, x0_e = 1.0 / math.sqrt(a_t), -math.sqrt(1.0 - a_t) / math.sqrt(a_t)
            else:
                x0_x, x0_e = math.sqrt(a_t), -math.sqrt(1.0 - a_t)
            d_x, d_e = c_out * x0_x + c_skip, c_out * x0_e
            st = StepPlan(t, d_x, d_e, [0.0] * 4, d_x, d_e, [0.0] * 4)
            if not last:
                st.cx, st.ce = math.sqrt(a_p) * d_x, math.sqrt(a_p) * d_e
                st.noise_scale, st.noise_offset = math.sqrt(1.0 - a_p), i
            out.append(st)
        return out


def lcm_scheduler_kwargs(config: dict) -> dict:
    """Constructor arguments of ``LCMScheduler`` from a checkpoint's ``scheduler_config.json``.  The options that make
    the step non-linear (sample clipping, dynamic thresholding) or change the beta table (zero-SNR rescaling, trained
    betas) raise a ValueError that names the key."""
    unsupported = {
        "clip_sample": bool,
        "thresholding": bool,
        "rescale_betas_zero_snr": bool,
        "trained_betas": lambda v: v is not None,
    }
    for key, bad in unsupported.items():
        if key in config and bad(config[key]):
            raise ValueError(f"scheduler config {key}={config[key]!r} is not supported by the LCM scheduler")
    if "prediction_type" in config:
        check_prediction_type(config["prediction_type"])
    used = ("original_inference_steps", "timestep_scaling", "prediction_type", "beta_start", "beta_end",
            "beta_schedule", "num_train_timesteps")
    return {key: config[key] for key in used if key in config}


SCHEDULER_MAP = {
    "DDIM": DDIMScheduler,
    "DPMSolverMultistep": DPMSolverMultistepScheduler,
    "PNDM": PNDMScheduler,
    "EulerDiscrete": EulerDiscreteScheduler,
    "EulerAncestralDiscrete": EulerAncestralDiscreteScheduler,
    "LMSDiscrete": LMSDiscreteScheduler,
    "LCM": LCMScheduler,
}

#: the scheduler classes whose loop state is y = x / sqrt(sigma^2 + 1)
SIGMA_SCHEDULERS = ("EulerDiscrete", "EulerAncestralDiscrete", "LMSDiscrete")


def sigma_scheduler_kwargs(config: dict) -> dict:
    """Constructor arguments of the Euler / Euler-ancestral / LMS samplers from a checkpoint's
    ``scheduler_config.json`` (the reference's ``SCHEDULER_MAP[name].from_config(pytorch_pipe.scheduler.config)``,
    pipeline.py:594-604, 672-676).  Settings these samplers do not implement raise a ValueError that names the key."""
    unsupported = {
        "prediction_type": lambda v: v not in (None, "epsilon"),
        "use_karras_sigmas": bool,
        "interpolation_type": lambda v: v not in (None, "linear"),
        "timestep_type": lambda v: v == "continuous",
        "rescale_betas_zero_snr": bool,
        "trained_betas": lambda v: v is not None,
    }
    for key, bad in unsupported.items():
        if key in config and bad(config[key]):
            raise ValueError(f"scheduler config {key}={config[key]!r} is not supported by the Euler / LMS samplers")
    used = ("timestep_spacing", "steps_offset", "beta_start", "beta_end", "beta_schedule", "num_train_timesteps")
    return {key: config[key] for key in used if key in config}


def make_scheduler(name, num_inference_steps, **kw):
    if name not in SCHEDULER_MAP:
        raise ValueError(f"unsupported scheduler {name!r}; available: {sorted(SCHEDULER_MAP)}")
    return SCHEDULER_MAP[name](num_inference_steps, **kw)


def apply_plan_host(step: StepPlan, guidance, eps_uncond, eps_text, x, hist, noise=None):
    """numpy mirror of the device kernel's arithmetic (host-logic tests only).  ``noise``: the step's normals z
    (needed when ``step.noise_offset >= 0``)."""
    eps = eps_uncond + guidance * (eps_text - eps_uncond)
    xp = step.cx * x + step.ce * eps
    x0 = step.x0_cx * x + step.x0_ce * eps
    for j in range(step.n_hist):
        xp = xp + step.ch[j] * hist[j]
        x0 = x0 + step.x0_ch[j] * hist[j]
    if step.noise_offset >= 0:
        if noise is None:
            raise ValueError("this step adds noise: pass its normals")
        xp = xp + step.noise_scale * noise
    if step.push_eps_slot >= 0:
        hist[step.push_eps_slot] = eps
    if step.push_x0_slot >= 0:
        hist[step.push_x0_slot] = x0
    if step.push_x_slot >= 0:
        hist[step.push_x_slot] = x
    return xp, x0
