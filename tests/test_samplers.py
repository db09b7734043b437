"""Host logic of the Euler, Euler-ancestral and LMS samplers: the y-space plans (y = x / sqrt(sigma^2 + 1), the UNet
input) must reproduce step-by-step restatements of diffusers 0.30.2 (tests/sampler_oracle.py) and the identities
between the samplers and DDIM.  No reference run pins these numerically; the identities below do."""
import dataclasses
import json
import math
import types

import numpy as np
import pytest
import torch
from scipy import integrate

import sampler_oracle as O
from b200sd import scheduler as S
from b200sd.rng import NvRandomSource
from oracle import restated as R

NAMES = ("EulerDiscrete", "EulerAncestralDiscrete", "LMSDiscrete")
SPACINGS = ("linspace", "leading", "trailing")


def _eps_fn(seed):
    rng = np.random.RandomState(seed)
    w = rng.randn(2)

    def f(x, t):
        base = np.tanh(x * 0.7 + t / 1000.0)
        return base * w[0] + 0.1, base * w[1] - 0.05
    return f


def test_sigma_table_and_timestep_pins():
    e = S.EulerDiscreteScheduler(20)
    assert abs(float(e.sigmas[0]) - 14.6146) < 1e-4 and abs(float(e.sigmas[-2]) - 0.029168) < 1e-6
    assert e.sigmas[-1] == 0 and e.sigmas.dtype == np.float32
    assert e.sigma_timesteps[0] == 999.0 and abs(e.sigma_timesteps[1] - 946.4211) < 1e-4
    assert e.timesteps[:4] == [999.0, 946.5, 894.0, 841.5]     # fp16-rounded, what the reference feeds the UNet
    assert abs(e.init_noise_sigma - 14.6146) < 1e-4
    le = S.EulerDiscreteScheduler(20, timestep_spacing="leading", steps_offset=1)
    assert le.sigma_timesteps[:2] == [951.0, 901.0] and le.sigma_timesteps[-1] == 1.0
    assert abs(float(le.sigmas[0]) - 11.0283) < 1e-4 and abs(le.init_noise_sigma - 11.0736) < 1e-4
    tr = S.EulerDiscreteScheduler(20, timestep_spacing="trailing")
    assert tr.sigma_timesteps[:2] == [999.0, 949.0] and tr.init_noise_sigma == float(tr.sigmas[0])
    for name in NAMES:
        for sp in SPACINGS:
            s, o = S.make_scheduler(name, 20, timestep_spacing=sp), O.ORACLES[name](20, timestep_spacing=sp)
            assert s.sigma_timesteps == o.timesteps
            np.testing.assert_allclose(s.sigmas, o.sigmas.numpy(), rtol=1e-6, atol=0)
            assert abs(s.init_noise_sigma - o.init_noise_sigma) < 2e-6 * o.init_noise_sigma
    with pytest.raises(ValueError):
        S.EulerDiscreteScheduler(20, timestep_spacing="bogus")
    with pytest.raises(ValueError):
        S.make_scheduler("Euler", 20)


@pytest.mark.parametrize("name", NAMES)
@pytest.mark.parametrize("spacing", SPACINGS)
@pytest.mark.parametrize("n", [1, 2, 4, 5, 20, 50])
def test_plans_match_the_oracle(name, spacing, n):
    """The y-space plan, applied with apply_plan_host and mapped back to x, reproduces diffusers' x-space steps."""
    s = S.make_scheduler(name, n, timestep_spacing=spacing)
    ref = O.ORACLES[name](n, timestep_spacing=spacing)
    plan = s.plan()
    assert len(plan) == len(ref.timesteps)
    assert [st.timestep for st in plan] == [float(np.float16(t)) for t in ref.timesteps]
    rng = np.random.RandomState(n)
    x = rng.randn(2, 4, 3, 3) * ref.init_noise_sigma
    f = _eps_fn(7)
    y = x / s.input_scale(0)
    hist = [np.zeros_like(x) for _ in range(4)]
    xr = torch.from_numpy(x.copy())
    src = NvRandomSource(1234)
    for i, st in enumerate(plan):
        # both sides see the same eps: the oracle's UNet input is scale_model_input(x)
        unet_in = ref.scale_model_input(xr, i).numpy()
        np.testing.assert_allclose(y, unet_in, rtol=1e-6, atol=1e-6 * np.abs(unet_in).max())
        eu, ec = f(unet_in, st.timestep)
        noise = None
        if st.noise_offset >= 0:
            src.offset = st.noise_offset
            noise = src.normal_array(x.size).reshape(x.shape)
        y, x0 = S.apply_plan_host(st, 7.5, eu, ec, y, hist, noise=noise)
        eps = torch.from_numpy(R.cfg_combine(eu, ec, 7.5))
        nz = torch.from_numpy(noise) if noise is not None else torch.zeros_like(xr)
        xr, x0r = O.oracle_step(ref, eps, xr, nz)
        x_plan = y * s.input_scale(i + 1)
        scale = max(1.0, float(xr.abs().max()))
        assert np.abs(x_plan - xr.numpy()).max() < 1e-6 * scale, (name, spacing, n, i)
        assert np.abs(x0 - x0r.numpy()).max() < 1e-6 * max(1.0, float(x0r.abs().max())), (name, spacing, n, i)
    assert s.input_scale(len(plan)) == 1.0     # the final sigma is 0: the loop state is the x-space latent


def _close(a, b, rel=1e-6):
    """max |a - b| within rel of the larger magnitude (DDIM's Swift-style fp32 table and diffusers' differ in the
    last bits)."""
    assert np.abs(a - b).max() <= rel * max(1.0, float(np.abs(b).max())), float(np.abs(a - b).max())


@pytest.mark.parametrize("n", [5, 20, 50])
def test_euler_leading_equals_ddim_until_the_last_step(n):
    """DDIM (eta 0) is the Euler step in sigma-space, x / sqrt(abar) = x0 + sigma eps: with the same 'leading' timesteps
    the UNet inputs agree and x' / sqrt(abar') agrees; the last Euler step lands on x0 (sigma' = 0)."""
    e = S.EulerDiscreteScheduler(n, timestep_spacing="leading", steps_offset=1).plan()
    d = S.DDIMScheduler(n).plan()
    assert [st.timestep for st in e] == [float(st.timestep) for st in d]
    abar = S.alphas_cumprod().astype(np.float64)
    es = S.EulerDiscreteScheduler(n, timestep_spacing="leading")
    rng = np.random.RandomState(0)
    x = rng.randn(3, 5)
    f = _eps_fn(2)
    y_e, x_d = x.copy(), x.copy()
    he, hd = [np.zeros_like(x) for _ in range(4)], [np.zeros_like(x) for _ in range(4)]
    for i in range(n):
        # DDIM's x_t and Euler's model input y_t are the same quantity: x_t = (x0 + sigma eps) sqrt(abar) = y_t
        _close(y_e, x_d)
        eu, ec = f(x_d, d[i].timestep)
        y_e, x0_e = S.apply_plan_host(e[i], 7.5, eu, ec, y_e, he)
        x_d, x0_d = S.apply_plan_host(d[i], 7.5, eu, ec, x_d, hd)
        _close(x0_e, x0_d)
        if i < n - 1:
            tp = d[i].timestep - 1000 // n
            x_e = y_e * es.input_scale(i + 1)
            _close(x_e, x_d / math.sqrt(abar[tp]))
        else:
            np.testing.assert_array_equal(y_e, x0_e)


@pytest.mark.parametrize("spacing", SPACINGS)
def test_lms_coefficients(spacing):
    lms = S.LMSDiscreteScheduler(20, timestep_spacing=spacing)
    eul = S.EulerDiscreteScheduler(20, timestep_spacing=spacing)
    # order 1 is the Euler step (LMS also stores its eps)
    assert dataclasses.replace(lms.plan()[0], push_eps_slot=-1) == eul.plan()[0]
    sig = lms.sigmas.astype(np.float64)
    for i in range(20):
        c = lms.lms_coefficients(i)
        assert len(c) == min(i + 1, 4)
        assert abs(sum(c) - (sig[i + 1] - sig[i])) < 1e-10 * abs(sig[i + 1] - sig[i]) + 1e-12
        order = len(c)
        for k in range(order):
            def basis(tau, k=k):
                p = 1.0
                for m in range(order):
                    if m != k:
                        p *= (tau - sig[i - m]) / (sig[i - k] - sig[i - m])
                return p
            q = integrate.quad(basis, sig[i], sig[i + 1], epsrel=1e-4)[0]
            assert abs(c[k] - q) < 1e-10 * max(1.0, abs(q)), (i, k)
        st = lms.plan()[i]
        s_next = lms.input_scale(i + 1)
        assert abs(st.ce * s_next - c[0]) < 1e-12 * max(1.0, abs(c[0]))
        assert st.push_eps_slot == i % 3 and st.n_hist == (3 if i else 0)
        for k in range(1, order):
            assert abs(st.ch[(i - k) % 3] * s_next - c[k]) < 1e-12 * max(1.0, abs(c[k]))


@pytest.mark.parametrize("spacing", SPACINGS)
def test_ancestral_identities(spacing):
    a = S.EulerAncestralDiscreteScheduler(20, timestep_spacing=spacing)
    eul = S.EulerDiscreteScheduler(20, timestep_spacing=spacing)
    sig = a.sigmas.astype(np.float64)
    plan = a.plan()
    for i, st in enumerate(plan):
        up, down = a.sigma_up_down(sig[i], sig[i + 1])
        assert abs(up ** 2 + down ** 2 - sig[i + 1] ** 2) < 1e-12 * max(1.0, sig[i + 1] ** 2)
        s_next = a.input_scale(i + 1)
        assert abs(st.noise_scale - up / s_next) < 1e-15
        # with zero noise the step is the Euler step to sigma_down
        e = eul.plan()[i]
        assert st.cx == e.cx and st.x0_cx == e.x0_cx and st.x0_ce == e.x0_ce
        assert abs(st.ce * s_next - (down - sig[i])) < 1e-12 * max(1.0, sig[i])
    assert [st.noise_offset for st in plan[:-1]] == list(range(19))
    assert plan[-1].noise_scale == 0.0 and plan[-1].noise_offset == -1
    for name in ("DDIM", "PNDM", "DPMSolverMultistep"):
        assert all(st.noise_scale == 0.0 and st.noise_offset == -1 for st in S.make_scheduler(name, 20).plan())
    with pytest.raises(ValueError, match="normals"):
        S.apply_plan_host(plan[0], 7.5, np.zeros(2), np.zeros(2), np.zeros(2), [np.zeros(2)] * 4)


def test_prepare_latents_scales_by_the_init_noise_sigma():
    from b200sd.pipeline import B200StableDiffusionPipeline as P

    stub = types.SimpleNamespace(vae_scale_factor=8)
    np.random.seed(3)
    base = P.prepare_latents(stub, 1, 4, 64, 64)
    for name in ("DDIM", "PNDM", "DPMSolverMultistep"):
        assert S.make_scheduler(name, 20).init_noise_sigma == 1.0
    for name in NAMES:
        for sp in SPACINGS:
            sigma = S.make_scheduler(name, 20, timestep_spacing=sp).init_noise_sigma
            np.random.seed(3)
            lat = P.prepare_latents(stub, 1, 4, 64, 64, init_noise_sigma=sigma)
            assert lat.dtype == np.float32
            np.testing.assert_array_equal(lat, base * np.float32(sigma))
    np.random.seed(3)
    np.testing.assert_array_equal(P.prepare_latents(stub, 1, 4, 64, 64, init_noise_sigma=1.0), base)


SDXL_SCHEDULER_CONFIG = {
    "_class_name": "EulerDiscreteScheduler", "_diffusers_version": "0.19.0.dev0", "beta_end": 0.012,
    "beta_schedule": "scaled_linear", "beta_start": 0.00085, "clip_sample": False, "interpolation_type": "linear",
    "num_train_timesteps": 1000, "prediction_type": "epsilon", "sample_max_value": 1.0, "set_alpha_to_one": False,
    "skip_prk_steps": True, "steps_offset": 1, "timestep_spacing": "leading", "trained_betas": None,
    "use_karras_sigmas": False,
}


def test_checkpoint_scheduler_config_mapping():
    kw = S.sigma_scheduler_kwargs(json.loads(json.dumps(SDXL_SCHEDULER_CONFIG)))
    assert kw == {"timestep_spacing": "leading", "steps_offset": 1, "beta_start": 0.00085, "beta_end": 0.012,
                  "beta_schedule": "scaled_linear", "num_train_timesteps": 1000}
    for name in NAMES:
        s = S.make_scheduler(name, 20, **kw)
        assert s.sigma_timesteps[:2] == [951.0, 901.0]
    # SD 2.1-base's config has no timestep_spacing key: the class default "linspace"
    assert S.sigma_scheduler_kwargs({"steps_offset": 1}) == {"steps_offset": 1}
    bad = [("prediction_type", "v_prediction"), ("use_karras_sigmas", True), ("interpolation_type", "log_linear"),
           ("timestep_type", "continuous"), ("rescale_betas_zero_snr", True), ("trained_betas", [0.1, 0.2])]
    for key, value in bad:
        with pytest.raises(ValueError, match=key):
            S.sigma_scheduler_kwargs(dict(SDXL_SCHEDULER_CONFIG, **{key: value}))
