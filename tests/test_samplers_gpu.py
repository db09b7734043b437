"""GPU tests of the Euler, Euler-ancestral and LMS samplers: the noised step kernel against its host twin
(rng.NvRandomSource), the device loop against the diffusers restatements (tests/sampler_oracle.py), the whole-loop CUDA
graph against the step-by-step path, and the checkpoint factory with SDXL's scheduler config."""
import json

import numpy as np
import pytest
import torch

import sampler_oracle as O
from b200sd import config
from b200sd import scheduler as S
from b200sd.rng import NvRandomSource
from oracle import restated as R

pytestmark = pytest.mark.gpu

NAMES = ("EulerDiscrete", "EulerAncestralDiscrete", "LMSDiscrete")


def _key(value):
    """A device Philox key holding the bits of the uint32 ``value``."""
    return torch.tensor([np.uint32(value).view(np.int32)], dtype=torch.int32, device="cuda")


def _coeffs(lib, st, guidance=7.5):
    from b200sd.pipeline import B200StableDiffusionPipeline as P
    return P._coeffs(st, guidance, lib.StepCoeffs())


@pytest.mark.parametrize("shape", [(1, 4, 64, 64), (8, 4, 64, 64), (2, 4, 17, 9)])
@pytest.mark.parametrize("key,offset", [(12345, 0), (0xDEADBEEF, 7), (2 ** 32 - 1, 2 ** 31 + 3)])
def test_noised_step_draws_the_nv_random_source_stream(cuda_lib, shape, key, offset):
    lib = cuda_lib
    n = shape[0]
    eps = torch.zeros(2 * n, *shape[1:], device="cuda")
    lat = torch.zeros(shape, device="cuda")
    k = lib.StepCoeffs()  # all coefficients 0
    k.push_eps_slot = k.push_x0_slot = k.push_x_slot = -1
    lib.cfg_scheduler_step_noised(eps, lat, k, 1.0, _key(key), offset)
    src = NvRandomSource(key)
    src.offset = offset
    want = src.normal_array(lat.numel()).reshape(shape)
    np.testing.assert_allclose(lat.cpu().numpy(), want, rtol=1e-5, atol=1e-5)
    again = torch.zeros(shape, device="cuda")
    lib.cfg_scheduler_step_noised(eps, again, k, 1.0, _key(key), offset)
    assert torch.equal(lat, again)


@pytest.mark.parametrize("name,step", [("LMSDiscrete", 5), ("PNDM", 3), ("DPMSolverMultistep", 4),
                                       ("EulerAncestralDiscrete", 2)])
def test_noised_step_with_zero_noise_equals_the_plain_step(cuda_lib, name, step):
    """noise_scale 0: the same latents, history pushes, denoised estimate and UNet input as b200sd_cfg_scheduler_step."""
    lib = cuda_lib
    n, c, h, w, c_pad = 2, 4, 16, 24, 8
    g = torch.Generator(device="cuda").manual_seed(step)
    eps = torch.randn(2 * n, c, h, w, device="cuda", generator=g)
    lat = torch.randn(n, c, h, w, device="cuda", generator=g)
    hist = torch.randn(4, n, c, h, w, device="cuda", generator=g)
    st = S.make_scheduler(name, 20).plan()[step]
    k = _coeffs(lib, st)
    outs = []
    for noised in (False, True):
        l, hh = lat.clone(), hist.clone()
        den = torch.empty_like(lat)
        unet_in = torch.zeros(2 * n, h, w, c_pad, dtype=torch.float16, device="cuda")
        if noised:
            lib.cfg_scheduler_step_noised(eps, l, k, 0.0, _key(99), 3, hist=hh, denoised=den, unet_in=unet_in)
        else:
            lib.cfg_scheduler_step(eps, l, k, hist=hh, denoised=den, unet_in=unet_in)
        outs.append((l, hh, den, unet_in))
    for a, b in zip(*outs):
        assert torch.equal(a, b)


def _tiny_pipe(name, spacing, **kw):
    from b200sd.pipeline import B200StableDiffusionPipeline
    pipe = B200StableDiffusionPipeline.from_random_init("tiny", images_per_call=2, height=64, width=64, seed=31,
                                                        scheduler=name, **kw)
    pipe.scheduler_kwargs = {"timestep_spacing": spacing}
    return pipe


@pytest.mark.parametrize("name", NAMES)
@pytest.mark.parametrize("spacing", ["linspace", "leading"])
def test_device_loop_vs_oracle(cuda_lib, name, spacing):
    """(a) the oracle sampler replayed on the engine's own noise predictions reproduces the recorded latents; (b) end to
    end against the all-oracle loop (the UNet's fp16 error grows by ~2g+1 per step under guidance)."""
    pipe = _tiny_pipe(name, spacing)
    prompts = ["a red cube", "a blue sphere"]
    steps, g, key = 5, 5.0, 77
    ref = O.ORACLES[name](steps, timestep_spacing=spacing)
    np.random.seed(5)
    lat0 = np.random.randn(2, 4, 16, 16).astype(np.float16).astype(np.float32) * np.float32(ref.init_noise_sigma)
    emb = pipe._encode_prompt(prompts, True, None)
    rec = []
    final = pipe.denoise(emb, lat0, steps, g, record=rec, noise_key=key).cpu().clone()
    src = NvRandomSource(key)

    def noise(i):
        src.offset = i
        return torch.from_numpy(src.normal_array(lat0.size).reshape(lat0.shape)).float()

    plan = S.make_scheduler(name, steps, timestep_spacing=spacing).plan()
    assert [r[0] for r in rec] == [st.timestep for st in plan] == [float(np.float16(t)) for t in ref.timesteps]
    # (a) scheduler + CFG kernel in isolation
    x = torch.from_numpy(lat0.copy())
    for i, (t, eps, lat_dev) in enumerate(rec):
        e = R.cfg_combine(eps[:2].cpu(), eps[2:].cpu(), g)
        x, _ = O.oracle_step(ref, e, x, noise(i))
        assert (lat_dev.cpu() - x).abs().max() < 2e-4 * max(1.0, float(x.abs().max())), (name, spacing, i)
    assert torch.equal(final, rec[-1][2].cpu())
    # (b) end to end
    ucfg = config.TINY_UNET
    usd = config.random_state_dict(config.unet_param_shapes(ucfg), seed=31, dtype=torch.float16)
    ref = O.ORACLES[name](steps, timestep_spacing=spacing)
    x = torch.from_numpy(lat0.copy())
    embt = torch.from_numpy(emb).float()
    with torch.no_grad():
        for i, t in enumerate(ref.timesteps):
            xin = ref.scale_model_input(torch.cat([x, x]), i).half().float()
            tt = torch.tensor([float(np.float16(t))] * 4)
            eps = R.unet_forward(usd, ucfg, xin, tt, embt)
            x, _ = O.oracle_step(ref, R.cfg_combine(eps[:2], eps[2:], g), x, noise(i))
    rel = float((final - x).abs().max() / x.abs().max())
    print(f"{name}/{spacing}: end-to-end latent rel err after {steps} steps = {rel:.3e}")
    assert rel < 5e-2, (name, spacing)


def test_ancestral_loop_graph_seeds_and_step_path(cuda_lib):
    pipe = _tiny_pipe("EulerAncestralDiscrete", "linspace")
    kw = dict(height=64, width=64, num_inference_steps=4, guidance_scale=5.0, output_type="np")
    prompts = ["a red cube", "a blue sphere"]
    a = pipe(prompts, seed=1, rng="nvidia", **kw).images
    assert pipe.loop_graph and len(pipe._loop_graphs) == 1
    b = pipe(prompts, seed=2, rng="nvidia", **kw).images
    assert len(pipe._loop_graphs) == 1            # the seed is not part of the graph key
    assert np.isfinite(a).all() and not np.array_equal(a, b)
    a2 = pipe(prompts, seed=1, rng="nvidia", **kw).images
    assert np.array_equal(a, a2)
    pipe.loop_graph = False
    a3 = pipe(prompts, seed=1, rng="nvidia", **kw).images
    pipe.loop_graph = True
    assert np.array_equal(a, a3), float(np.abs(a - a3).max())
    # without a seed the key comes from the global numpy stream, right after the latents
    np.random.seed(11)
    c = pipe(prompts, **kw).images
    np.random.seed(11)
    assert np.array_equal(c, pipe(prompts, **kw).images)
    # the numpy source keys the noise with the seed at draw numbers 0, 1, ...; the nvidia source continues after the
    # latents' two draws
    n1 = pipe(prompts, seed=1, rng="numpy", **kw).images
    assert np.isfinite(n1).all() and len(pipe._loop_graphs) == 2


def test_controlnet_euler_graph_equals_eager(cuda_lib):
    from b200sd.pipeline import B200StableDiffusionPipeline
    pipe = B200StableDiffusionPipeline.from_random_init("tiny", images_per_call=1, height=64, width=64, seed=21,
                                                        controlnet_cfgs=[config.TINY_CONTROLNET],
                                                        scheduler="EulerDiscrete")
    np.random.seed(5)
    cond = np.random.rand(3, 128, 128).astype(np.float16)
    kw = dict(height=64, width=64, num_inference_steps=4, guidance_scale=5.0, output_type="np", seed=3,
              controlnet_cond=[cond])
    a = pipe("a cat", **kw).images
    assert len(pipe._loop_graphs) == 1
    pipe.loop_graph = False
    b = pipe("a cat", **kw).images
    pipe.loop_graph = True
    assert np.isfinite(a).all() and np.array_equal(a, b), float(np.abs(a - b).max())


def test_image_to_image_is_refused(cuda_lib):
    pipe = _tiny_pipe("LMSDiscrete", "linspace")
    with pytest.raises(ValueError, match="image-to-image"):
        pipe(["a", "b"], height=64, width=64, num_inference_steps=2, starting_image=np.zeros((2, 3, 64, 64)))


def test_from_pretrained_with_sdxl_euler_config(cuda_lib, tmp_path):
    from test_factory_gpu import _model_dir
    from test_samplers import SDXL_SCHEDULER_CONFIG
    from b200sd.pipeline import B200StableDiffusionPipeline

    _model_dir(tmp_path, config.TINY_XL_UNET, seed=51)
    (tmp_path / "scheduler" / "scheduler_config.json").write_text(json.dumps(SDXL_SCHEDULER_CONFIG))
    with pytest.raises(ValueError, match="EulerDiscrete"):
        B200StableDiffusionPipeline.from_pretrained(str(tmp_path), height=64, width=64)
    pipe = B200StableDiffusionPipeline.from_pretrained(str(tmp_path), height=64, width=64,
                                                       scheduler_override="EulerDiscrete")
    assert pipe.xl and pipe.scheduler_name == "EulerDiscrete"
    sched = S.make_scheduler(pipe.scheduler_name, 5, **pipe.scheduler_kwargs)
    assert sched.timestep_spacing == "leading" and sched.steps_offset == 1
    assert sched.timesteps == [801.0, 601.0, 401.0, 201.0, 1.0]
    g = torch.Generator().manual_seed(3)
    emb = torch.randn(2, 96, 1, 77, generator=g).half().numpy()
    pooled = torch.randn(2, 64, generator=g).numpy()
    img = pipe("x", height=64, width=64, num_inference_steps=5, guidance_scale=4.0, output_type="np", seed=4,
               prompt_embeds=emb, pooled_prompt_embeds=pooled).images
    assert img.shape == (1, 64, 64, 3) and np.isfinite(img).all()
    bad = dict(SDXL_SCHEDULER_CONFIG, prediction_type="v_prediction")
    (tmp_path / "scheduler" / "scheduler_config.json").write_text(json.dumps(bad))
    with pytest.raises(ValueError, match="prediction_type"):
        B200StableDiffusionPipeline.from_pretrained(str(tmp_path), height=64, width=64,
                                                    scheduler_override="EulerAncestralDiscrete")
