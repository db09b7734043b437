"""v-prediction (SD 2.0 / 2.1 768-v) in the DDIM, DPM-Solver++ and PNDM plans: step by step against the restatements of
diffusers 0.30.2 (tests/vpred_oracle.py), the identities that tie a v-plan to the epsilon plan, the SD21_UNET config,
and the restated UNet against the reference's own output at 96x96 latents (tests/golden/make_golden_sd21_768.py)."""
import json
import math
import os

import numpy as np
import pytest
import torch

import vpred_oracle as V
from b200sd import config
from b200sd import scheduler as S
from oracle import restated as R

GOLD = os.path.join(os.path.dirname(__file__), "golden")
NAMES = ("DDIM", "DPMSolverMultistep", "PNDM")
ABAR = R.alphas_cumprod()


def _sched(name, n, **kw):
    s = S.make_scheduler(name, n, **kw)
    s.abar = ABAR.double().numpy()  # the oracle's fp32 table on both sides
    return s


def _model(seed):
    """A smooth stand-in for the UNet: (uncond, cond) outputs from the latents and the timestep."""
    w = np.random.RandomState(seed).randn(2)

    def f(x, t):
        base = np.tanh(x * 0.7 + t / 1000.0)
        return base * w[0] + 0.1, base * w[1] - 0.05
    return f


def _run_plan(sched, fn, x0, guidance=7.5, start=0):
    x, hist = x0.copy(), [np.zeros_like(x0) for _ in range(4)]
    xs, x0s, outs = [], [], []
    for st in sched.plan(start=start):
        eu, ec = fn(x, st.timestep)
        outs.append(eu + guidance * (ec - eu))
        x, den = S.apply_plan_host(st, guidance, eu, ec, x, hist)
        xs.append(x.copy())
        x0s.append(den.copy())
    return xs, x0s, outs


def _cases():
    for name in NAMES:
        for n in (1, 2, 3, 4, 5, 10, 14, 15, 20, 25, 50):
            for kw in ([{"final_sigmas_type": "zero"}, {"final_sigmas_type": "sigma_min"}]
                       if name == "DPMSolverMultistep" else [{}]):
                for start in sorted({0, n // 2, n - 1}):
                    yield name, n, kw, start


@pytest.mark.parametrize("name,n,kw,start", list(_cases()))
def test_vpred_plans_match_the_diffusers_restatement(name, n, kw, start):
    sched = _sched(name, n, prediction_type="v_prediction", **kw)
    ref = V.ORACLES[name](n, start=start, abar=ABAR, **kw)
    assert [st.timestep for st in sched.plan(start=start)] == ref.timesteps
    x = np.random.RandomState(n).randn(2, 4, 6, 6)
    fn = _model(n + start)
    xs, x0s, _ = _run_plan(sched, fn, x, start=start)
    xr = torch.from_numpy(x.copy())
    for i, t in enumerate(ref.timesteps):
        eu, ec = fn(xr.numpy(), t)
        xr, x0r = ref.step(torch.from_numpy(R.cfg_combine(eu, ec, 7.5)), xr)
        scale = max(1.0, float(xr.abs().max()))
        assert np.abs(xs[i] - xr.numpy()).max() <= 1e-6 * scale, (name, n, kw, start, i)
        assert np.abs(x0s[i] - x0r.numpy()).max() <= 1e-6 * max(1.0, float(x0r.abs().max())), (name, n, kw, start, i)


@pytest.mark.parametrize("name,kw", [("DDIM", {}), ("DPMSolverMultistep", {"final_sigmas_type": "zero"}),
                                     ("DPMSolverMultistep", {"final_sigmas_type": "sigma_min"})])
@pytest.mark.parametrize("n,start", [(1, 0), (5, 0), (14, 0), (20, 0), (50, 0), (20, 10), (14, 9)])
def test_vpred_plan_reproduces_the_epsilon_trajectory(name, kw, n, start):
    """Feed the v-plan v_k = alpha_t eps_k - sigma_t x0_k built from the epsilon plan's own trajectory: DDIM and
    DPM-Solver++ work on (x0, eps) pairs, so both plans must produce the same latents and x0 at every step."""
    eps_plan = S.make_scheduler(name, n, **kw)
    xs, x0s, eps = _run_plan(eps_plan, _model(7), np.random.RandomState(3).randn(2, 4, 6, 6), guidance=1.0,
                             start=start)
    v_plan = S.make_scheduler(name, n, prediction_type="v_prediction", **kw)
    abar = v_plan.abar
    vs = [math.sqrt(abar[st.timestep]) * e - math.sqrt(1 - abar[st.timestep]) * x0
          for st, e, x0 in zip(v_plan.plan(start=start), eps, x0s)]
    k = iter(vs)
    xv, x0v, _ = _run_plan(v_plan, lambda x, t: (np.zeros_like(x), next(k)), np.random.RandomState(3).randn(2, 4, 6, 6),
                           guidance=1.0, start=start)
    for i in range(len(xs)):
        assert np.abs(xv[i] - xs[i]).max() <= 1e-12 * max(1.0, np.abs(xs[i]).max()), (name, kw, n, start, i)
        assert np.abs(x0v[i] - x0s[i]).max() <= 1e-12 * max(1.0, np.abs(x0s[i]).max()), (name, kw, n, start, i)


@pytest.mark.parametrize("n", [3, 10, 20])
def test_pndm_vpred_first_step_is_the_epsilon_step(n):
    """On its first step PLMS converts the current v with the current sample, so it equals the epsilon step fed
    eps = alpha_t v + sigma_t x."""
    x = np.random.RandomState(n).randn(2, 4, 6, 6)
    v = np.random.RandomState(n + 1).randn(2, 4, 6, 6)
    vst = S.PNDMScheduler(n, prediction_type="v_prediction").plan()[0]
    est = S.PNDMScheduler(n).plan()[0]
    abar = S.PNDMScheduler(n).abar[vst.timestep]
    e = math.sqrt(abar) * v + math.sqrt(1 - abar) * x
    zero = np.zeros_like(x)
    xv, x0v = S.apply_plan_host(vst, 1.0, zero, v, x, [zero.copy() for _ in range(4)])
    xe, x0e = S.apply_plan_host(est, 1.0, zero, e, x, [zero.copy() for _ in range(4)])
    assert np.abs(xv - xe).max() <= 1e-12 and np.abs(x0v - x0e).max() <= 1e-12


def test_pndm_vpred_three_steps_evaluated_by_hand():
    """PLMS with v, 3 inference steps (4 model calls), written out from diffusers' _get_prev_sample: the ring keeps the
    raw outputs; each step combines them into e with the Adams-Bashforth weights, then moves with the sample s and the
    (shifted) timestep t as x' = (sc + mc sigma_t) s + mc alpha_t e, x0 = alpha_t s - sigma_t e."""
    n, d = 3, 1000 // 3
    s = S.PNDMScheduler(n, prediction_type="v_prediction")
    ts = s.timesteps
    assert ts == [667, 334, 334, 1]
    abar = np.cumprod(1.0 - np.linspace(0.00085 ** 0.5, 0.012 ** 0.5, 1000, dtype=np.float64) ** 2)
    s.abar = abar

    def step(x, t, tp, e):
        a_t, a_p = abar[t], abar[max(0, tp)]
        sc = np.sqrt(a_p / a_t)
        mc = -(a_p - a_t) / (a_t * np.sqrt(1 - a_p) + np.sqrt(a_t * (1 - a_t) * a_p))
        al, sg = np.sqrt(a_t), np.sqrt(1 - a_t)
        return (sc + mc * sg) * x + mc * al * e, al * x - sg * e

    rng = np.random.RandomState(0)
    x0 = rng.randn(3, 5)
    vs = [rng.randn(3, 5) for _ in range(4)]
    k = iter(vs)
    xs, dens, _ = _run_plan(s, lambda x, t: (np.zeros_like(x), next(k)), x0, guidance=1.0)
    x1, d1 = step(x0, 667, 667 - d, vs[0])                          # counter 0: saves x0
    x2, d2 = step(x0, 667, 334, 0.5 * (vs[1] + vs[0]))               # counter 1: from the saved sample, t shifted back
    x3, d3 = step(x2, 334, 1, 1.5 * vs[2] - 0.5 * vs[0])             # ring [v0, v2] (v1 is not stored)
    x4, d4 = step(x3, 1, 1 - d, (23 * vs[3] - 16 * vs[2] + 5 * vs[0]) / 12)
    want = [(x1, d1), (x2, d2), (x3, d3), (x4, d4)]
    for i, (wx, wd) in enumerate(want):
        assert np.allclose(xs[i], wx, rtol=1e-12, atol=1e-12), i
        assert np.allclose(dens[i], wd, rtol=1e-12, atol=1e-12), i
    # the epsilon sampler fed the converted outputs differs after the first step
    ab = [abar[667], abar[667], abar[334], abar[1]]
    samples = [x0, x0, x2, x3]
    k = iter([np.sqrt(a) * v + np.sqrt(1 - a) * smp for a, v, smp in zip(ab, vs, samples)])
    e_plan = S.PNDMScheduler(n)
    e_plan.abar = abar
    xe, _, _ = _run_plan(e_plan, lambda x, t: (np.zeros_like(x), next(k)), x0, guidance=1.0)
    assert np.allclose(xe[0], xs[0], rtol=1e-12, atol=1e-12) and not np.allclose(xe[2], xs[2], rtol=1e-6, atol=1e-6)


@pytest.mark.parametrize("name", NAMES)
def test_epsilon_is_the_default(name):
    kws = [{"final_sigmas_type": "zero"}, {}] if name == "DPMSolverMultistep" else [{}]
    for kw in kws:
        for n, start in ((1, 0), (7, 0), (20, 0), (20, 10), (50, 49)):
            assert (S.make_scheduler(name, n, prediction_type="epsilon", **kw).plan(start=start)
                    == S.make_scheduler(name, n, **kw).plan(start=start))
    assert S.make_scheduler(name, 20).prediction_type == "epsilon"


@pytest.mark.parametrize("name", NAMES)
@pytest.mark.parametrize("value", ["sample", "v-prediction", "", None])
def test_unsupported_prediction_types_raise(name, value):
    with pytest.raises(ValueError, match="prediction_type"):
        S.make_scheduler(name, 20, prediction_type=value)


def test_sigma_schedulers_keep_refusing_v_prediction():
    with pytest.raises(ValueError, match="prediction_type"):
        S.sigma_scheduler_kwargs({"prediction_type": "v_prediction"})
    with pytest.raises(TypeError):
        S.make_scheduler("EulerDiscrete", 20, prediction_type="v_prediction")


# the stabilityai/stable-diffusion-2-1 unet/config.json (diffusers 0.10.0.dev0)
SD21_UNET_CONFIG = {
    "_class_name": "UNet2DConditionModel", "_diffusers_version": "0.10.0.dev0", "act_fn": "silu",
    "attention_head_dim": [5, 10, 20, 20], "block_out_channels": [320, 640, 1280, 1280], "center_input_sample": False,
    "cross_attention_dim": 1024,
    "down_block_types": ["CrossAttnDownBlock2D", "CrossAttnDownBlock2D", "CrossAttnDownBlock2D", "DownBlock2D"],
    "downsample_padding": 1, "dual_cross_attention": False, "flip_sin_to_cos": True, "freq_shift": 0, "in_channels": 4,
    "layers_per_block": 2, "mid_block_scale_factor": 1, "norm_eps": 1e-05, "norm_num_groups": 32,
    "num_class_embeds": None, "only_cross_attention": False, "out_channels": 4, "sample_size": 96,
    "up_block_types": ["UpBlock2D", "CrossAttnUpBlock2D", "CrossAttnUpBlock2D", "CrossAttnUpBlock2D"],
    "upcast_attention": True, "use_linear_projection": True,
}


def test_sd21_config_and_checkpoint_config(tmp_path):
    """SD21_UNET is the SD-2.1-base UNet at 96x96 latents, and the checkpoint's config.json reads into the same
    architecture (upcast_attention / use_linear_projection are what the engine does anyway)."""
    from b200sd import checkpoint as K
    assert config.SD21_UNET == dict(config.SD21_BASE_UNET, sample_size=96)
    os.makedirs(tmp_path / "unet")
    (tmp_path / "unet" / "config.json").write_text(json.dumps(SD21_UNET_CONFIG))
    cfg = K.read_config(str(tmp_path), "unet")
    assert cfg["upcast_attention"] is True and cfg["use_linear_projection"] is True
    assert set(config.SD21_UNET) - set(cfg) == {"transformer_layers_per_block"}  # diffusers' default: 1
    for key, value in config.SD21_UNET.items():
        assert cfg.get(key, 1) == value, key
    assert config.unet_param_shapes(cfg) == config.unet_param_shapes(config.SD21_UNET)
    # a linear proj_in / proj_out ([out, in], use_linear_projection) passes the schema check
    shapes = config.unet_param_shapes(config.SD21_UNET)
    sd = {k: torch.empty(v[:2] if k.endswith(("proj_in.weight", "proj_out.weight")) else v, dtype=torch.float16)
          for k, v in shapes.items()}
    assert len(K.check_state_dict("unet", cfg, sd)) == len(shapes)


def test_restated_unet_matches_reference_golden_sd21_768():
    gold = np.load(os.path.join(GOLD, "unet_sd21_768.npz"))
    cfg = config.SD21_UNET
    sd = config.random_state_dict(config.unet_param_shapes(cfg), seed=int(gold["weight_seed"]))
    keys = sorted(sd.keys())
    fp = np.array([float(sd[k].double().sum()) for k in (keys[0], keys[len(keys) // 2], keys[-1])] + [float(len(keys))])
    assert np.allclose(fp, gold["fingerprint"], rtol=1e-6), "weight generator drifted"
    g = torch.Generator().manual_seed(int(gold["input_seed"]))
    x = torch.randn(2, 4, 96, 96, generator=g)
    c = torch.randn(2, 1024, 1, 77, generator=g)
    with torch.no_grad():
        y = R.unet_forward(sd, cfg, x, torch.tensor([float(gold["timestep"])] * 2), c).numpy()
    ref = gold["noise_pred_ORIGINAL"]
    assert y.shape == ref.shape == (2, 4, 96, 96)
    assert np.abs(y - ref).max() < 2e-5
    assert R.compute_psnr(torch.from_numpy(y), torch.from_numpy(ref)) > 100
