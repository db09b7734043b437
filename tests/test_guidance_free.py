"""Host-side tests of the guidance-free loop, guidance-embedding (LCM) UNets and the LCM scheduler: the LCM timesteps
and step plans against a numpy restatement of diffusers 0.30.2's formulas, its scheduler-config reader, the guidance
embedding, the UNet schema's cond_proj, the CFG rule, from_pretrained's scheduler classes and every new ValueError.

``unet_forward_cond`` is the CPU oracle of a guidance-embedding UNet: oracle.restated's UNet with
cond_proj(timestep_cond) added to the sinusoidal embedding before time_embedding.linear_1, pinned here to the
reference's own ``TimestepEmbedding(cond_proj_dim=...)``."""
import contextlib
import types

import numpy as np
import pytest
import torch

from b200sd import config
from b200sd import scheduler as S
from b200sd.pipeline import B200StableDiffusionPipeline as P
from b200sd.unet import guidance_scale_embedding
from oracle import restated as R

_PLAIN_TIME_MLP = R._time_mlp


def time_mlp_cond(sd, prefix, x, cond):
    """TimestepEmbedding.forward with a condition: linear_2(silu(linear_1(x + cond_proj(cond))))."""
    x = x + R._conv(sd, prefix + ".cond_proj", R._f(cond)[:, :, None, None])[:, :, 0, 0]
    return _PLAIN_TIME_MLP(sd, prefix, x)


@contextlib.contextmanager
def _time_condition(cond):
    def mlp(sd, prefix, x):
        return time_mlp_cond(sd, prefix, x, cond) if prefix == "time_embedding" else _PLAIN_TIME_MLP(sd, prefix, x)
    R._time_mlp = mlp
    try:
        yield
    finally:
        R._time_mlp = _PLAIN_TIME_MLP


def unet_forward_cond(sd, cfg, sample, timestep, encoder_hidden_states, timestep_cond, **kw):
    """oracle.restated.unet_forward of a guidance-embedding UNet (``time_cond_proj_dim``)."""
    with _time_condition(timestep_cond):
        return R.unet_forward(sd, cfg, sample, timestep, encoder_hidden_states, **kw)


# ---------------------------------------------------------------------------------------------------------- LCM
def _lcm_numpy(n, prediction_type, x, eps, zs, original_steps=50, scaling=10.0):
    """diffusers 0.30.2 LCMScheduler.set_timesteps + step, restated in numpy float64 (noise zs[i] on step i)."""
    abar = S.alphas_cumprod_diffusers().astype(np.float64)
    k = 1000 // original_steps
    origin = (np.arange(1, original_steps + 1) * k - 1)[::-1]
    ts = origin[np.floor(np.linspace(0, len(origin), n, endpoint=False)).astype(np.int64)]
    outs = []
    for i, t in enumerate(ts):
        prev = ts[i + 1] if i + 1 < len(ts) else t
        a_t, a_p = abar[t], abar[prev]
        s = t * scaling
        c_skip, c_out = 0.25 / (s ** 2 + 0.25), s / np.sqrt(s ** 2 + 0.25)
        if prediction_type == "epsilon":
            x0 = (x - np.sqrt(1 - a_t) * eps[i]) / np.sqrt(a_t)
        else:
            x0 = np.sqrt(a_t) * x - np.sqrt(1 - a_t) * eps[i]
        den = c_out * x0 + c_skip * x
        x = np.sqrt(a_p) * den + np.sqrt(1 - a_p) * zs[i] if i < len(ts) - 1 else den
        outs.append((int(t), x, den))
    return outs


def test_lcm_timesteps_known_answers():
    assert S.LCMScheduler(4).timesteps == [999, 759, 499, 259]
    assert S.LCMScheduler(8).timesteps == [999, 879, 759, 639, 499, 379, 259, 139]
    assert S.LCMScheduler(1).timesteps == [999]
    assert S.LCMScheduler(50).timesteps == list(range(999, 0, -20))


@pytest.mark.parametrize("prediction_type", ["epsilon", "v_prediction"])
@pytest.mark.parametrize("n,seed", [(1, 0), (4, 1), (8, 2)])
def test_lcm_plan_matches_the_formulas(prediction_type, n, seed):
    rs = np.random.RandomState(seed)
    x0 = rs.standard_normal((2, 4, 3, 5))
    eps = rs.standard_normal((n, 2, 4, 3, 5))
    zs = rs.standard_normal((n, 2, 4, 3, 5))
    want = _lcm_numpy(n, prediction_type, x0, eps, zs)
    plan = S.LCMScheduler(n, prediction_type=prediction_type).plan()
    x = x0
    for i, (st, (t, x_next, den)) in enumerate(zip(plan, want)):
        assert st.timestep == t
        hist = np.zeros((4,) + x.shape)
        noise = zs[i] if st.noise_offset >= 0 else None
        xp, d = S.apply_plan_host(st, 1.0, eps[i], eps[i], x, hist, noise)
        np.testing.assert_allclose(d, den, rtol=1e-10, atol=1e-10)
        np.testing.assert_allclose(xp, x_next, rtol=1e-10, atol=1e-10)
        if i == n - 1:
            assert st.noise_offset == -1 and st.noise_scale == 0.0   # the last step lands on the denoised estimate
        else:
            assert st.noise_offset == i
        x = xp


def test_lcm_scheduler_kwargs_reads_a_typical_config():
    cfg = {"_class_name": "LCMScheduler", "_diffusers_version": "0.22.0.dev0", "beta_end": 0.012,
           "beta_schedule": "scaled_linear", "beta_start": 0.00085, "clip_sample": False, "clip_sample_range": 1.0,
           "dynamic_thresholding_ratio": 0.995, "num_train_timesteps": 1000, "original_inference_steps": 50,
           "prediction_type": "epsilon", "rescale_betas_zero_snr": False, "sample_max_value": 1.0,
           "set_alpha_to_one": True, "steps_offset": 1, "thresholding": False, "timestep_scaling": 10.0,
           "timestep_spacing": "leading", "trained_betas": None}
    kw = S.lcm_scheduler_kwargs(cfg)
    assert kw == {"original_inference_steps": 50, "timestep_scaling": 10.0, "prediction_type": "epsilon",
                  "beta_start": 0.00085, "beta_end": 0.012, "beta_schedule": "scaled_linear",
                  "num_train_timesteps": 1000}
    assert S.make_scheduler("LCM", 4, **kw).timesteps == [999, 759, 499, 259]


@pytest.mark.parametrize("key,value", [("clip_sample", True), ("thresholding", True), ("rescale_betas_zero_snr", True),
                                       ("trained_betas", [0.1] * 1000)])
def test_lcm_scheduler_kwargs_rejects_nonlinear_options(key, value):
    with pytest.raises(ValueError, match=key):
        S.lcm_scheduler_kwargs({key: value})


def test_lcm_scheduler_errors():
    with pytest.raises(ValueError, match="original_inference_steps"):
        S.LCMScheduler(51)
    with pytest.raises(ValueError, match="prediction_type"):
        S.LCMScheduler(4, prediction_type="sample")
    with pytest.raises(ValueError, match="image-to-image"):
        S.LCMScheduler(4).plan(start=1)


# ----------------------------------------------------------------------------------------- guidance embedding
@pytest.mark.parametrize("g,d", [(8.5, 256), (1.0, 256), (4.0, 255), (0.0, 64)])
def test_guidance_embedding_formula(g, d):
    emb = guidance_scale_embedding(g, d, batch=3)
    assert emb.shape == (3, d) and emb.dtype == torch.float32 and torch.equal(emb[0], emb[2])
    half = d // 2
    w = (g - 1.0) * 1000.0
    f = np.exp(-np.arange(half) * np.log(10000.0) / (half - 1))
    want = np.concatenate([np.sin(w * f), np.cos(w * f), np.zeros(d % 2)])
    np.testing.assert_allclose(emb[0].numpy(), want, atol=2e-3 * max(1.0, abs(w) / 1000))
    if g == 1.0:  # w = 0: [0 ... 0, 1 ... 1]
        assert torch.equal(emb[0], torch.cat([torch.zeros(half), torch.ones(half)]))
    if d % 2:
        assert emb[0, -1] == 0


# ------------------------------------------------------------------------------------------------- UNet schema
@pytest.mark.parametrize("dim", [None, 0, 256])
def test_schema_includes_cond_proj_exactly_when_set(dim):
    cfg = dict(config.SD15_UNET, time_cond_proj_dim=dim)
    sh = config.unet_param_shapes(cfg)
    if dim:
        assert sh["time_embedding.cond_proj.weight"] == (320, 256, 1, 1)
        assert "time_embedding.cond_proj.bias" not in sh
        assert set(sh) - set(config.unet_param_shapes(config.SD15_UNET)) == {"time_embedding.cond_proj.weight"}
    else:
        assert sh == config.unet_param_shapes(config.SD15_UNET)


def test_check_state_dict_requires_cond_proj():
    from b200sd import checkpoint as K
    cfg = dict(config.TINY_UNET, time_cond_proj_dim=16)
    sd = config.random_state_dict(config.unet_param_shapes(cfg), seed=0)
    sd["time_embedding.cond_proj.weight"] = sd["time_embedding.cond_proj.weight"][:, :, 0, 0]  # the Linear shape
    assert "time_embedding.cond_proj.weight" in K.check_state_dict("unet", cfg, sd)
    del sd["time_embedding.cond_proj.weight"]
    with pytest.raises(KeyError):
        K.check_state_dict("unet", cfg, sd)


def test_oracle_time_embedding_pinned_to_reference_class():
    from oracle import ref_unet
    if not ref_unet.available():
        pytest.skip("reference tree not available")
    unet_mod = ref_unet.load().unet
    torch.manual_seed(0)
    ref = unet_mod.TimestepEmbedding(32, 128, cond_proj_dim=24).eval()
    sd = {f"time_embedding.{k}": v for k, v in ref.state_dict().items()}
    t_emb = torch.randn(3, 32)
    cond = torch.randn(3, 24)
    with torch.no_grad():
        want = ref(t_emb, cond).reshape(3, -1)
        got = time_mlp_cond(sd, "time_embedding", t_emb, cond).reshape(3, -1)
    assert torch.allclose(got, want, atol=1e-5), float((got - want).abs().max())


def test_oracle_unet_with_cond_reduces_to_the_plain_one_for_a_zero_projection():
    cfg = dict(config.TINY_UNET, time_cond_proj_dim=8)
    sd = config.random_state_dict(config.unet_param_shapes(cfg), seed=3)
    x = torch.randn(1, 4, 16, 16)
    c = torch.randn(1, cfg["cross_attention_dim"], 1, 77)
    t = torch.tensor([501.0])
    cond = guidance_scale_embedding(8.0, 8)
    with torch.no_grad():
        y = unet_forward_cond(sd, cfg, x, t, c, cond)
        sd0 = dict(sd, **{"time_embedding.cond_proj.weight": torch.zeros_like(sd["time_embedding.cond_proj.weight"])})
        y0 = unet_forward_cond(sd0, cfg, x, t, c, cond)
        plain = R.unet_forward(sd, cfg, x, t, c)
    assert torch.equal(y0, plain) and not torch.allclose(y, plain)
    assert R._time_mlp is _PLAIN_TIME_MLP  # the context restored the oracle


# ------------------------------------------------------------------------------------------------ pipeline rules
def _stub(time_cond_dim=0, **kw):
    unet = types.SimpleNamespace(engine=types.SimpleNamespace(time_cond_dim=time_cond_dim), batch=2)
    s = types.SimpleNamespace(unet=unet, **kw)
    s.do_classifier_free_guidance = lambda g: P.do_classifier_free_guidance(s, g)
    return s


@pytest.mark.parametrize("g", [0.0, 0.5, 1.0, 1.0001, 7.5])
@pytest.mark.parametrize("dim", [0, 256])
def test_cfg_rule(g, dim):
    assert P.do_classifier_free_guidance(_stub(dim), g) == (g > 1.0 and dim == 0)


def test_from_pretrained_scheduler_class_map():
    want = {"PNDMScheduler": "PNDM", "DDIMScheduler": "DDIM", "DPMSolverMultistepScheduler": "DPMSolverMultistep",
            "LCMScheduler": "LCM", "EulerDiscreteScheduler": "EulerDiscrete",
            "EulerAncestralDiscreteScheduler": "EulerAncestralDiscrete", "LMSDiscreteScheduler": "LMSDiscrete"}
    assert P._SCHEDULER_CLASS == want
    assert set(want.values()) <= set(S.SCHEDULER_MAP)
    for cls, name in want.items():
        cfg = {"_class_name": cls, "timestep_spacing": "trailing"}
        assert P.scheduler_from_config(cfg) == name
        if name in S.SIGMA_SCHEDULERS:  # other spacings (SDXL-base's "leading" Euler) still need scheduler_override
            for sp in ("leading", "linspace", None):
                with pytest.raises(ValueError, match="scheduler_override"):
                    P.scheduler_from_config({"_class_name": cls, "timestep_spacing": sp})
        else:
            assert P.scheduler_from_config({"_class_name": cls, "timestep_spacing": "leading"}) == name
    assert P.scheduler_from_config({}) == "PNDM"
    with pytest.raises(ValueError, match="KDPM2DiscreteScheduler.*not implemented"):
        P.scheduler_from_config({"_class_name": "KDPM2DiscreteScheduler"})


@pytest.mark.parametrize("arg", ["starting_image", "mask_image"])
def test_lcm_rejects_image_inputs(arg):
    s = _stub(256, height=64, width=64, controlnet=None, images_per_call=1, scheduler_name="LCM")
    s.check_inputs = lambda *a: P.check_inputs(s, *a)
    kw = {"starting_image": np.zeros((1, 3, 64, 64), np.float32)}
    if arg == "mask_image":
        kw["mask_image"] = np.ones((64, 64), np.float32)
    with pytest.raises(ValueError, match=arg):
        P.__call__(s, "x", height=64, width=64, num_inference_steps=4, guidance_scale=8.0, **kw)


def test_refiner_needs_guidance():
    s = _stub(0, scheduler_name="DDIM", scheduler_kwargs={}, images_per_call=1)
    with pytest.raises(ValueError, match="refiner"):
        P.denoise(s, np.zeros((2, 8, 1, 77)), np.zeros((1, 4, 8, 8)), 4, 1.0, refiner={})


def test_capi_rejects_time_condition():
    from b200sd import capi
    with pytest.raises(ValueError, match="time_cond_proj_dim"):
        capi.make_config(dict(config.TINY_UNET, time_cond_proj_dim=256), 2, 16, 16)
