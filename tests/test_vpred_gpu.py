"""GPU tests of Stable Diffusion 2.0 / 2.1 768-v: the SD-2.1 UNet at 96x96 latents against the reference's output
(tests/golden/make_golden_sd21_768.py), every GEMM / convolution launch of it against an fp32 reference of that launch,
level-0 self-attention over 9216 tokens under both attention schedules, and v-prediction in the DDIM, DPM-Solver++
and PNDM device loops against the diffusers restatements (tests/vpred_oracle.py), through to ``from_pretrained``."""
import json
import os

import numpy as np
import pytest
import torch

import vpred_oracle as V
from b200sd import config
from b200sd import scheduler as S
from oracle import restated as R
from model_cases import model_inputs as _model_inputs
from test_gemm_plans_gpu import _Replay
from test_unet_gpu import _check

pytestmark = pytest.mark.gpu
GOLD = os.path.join(os.path.dirname(__file__), "golden")
CASES = [("DDIM", {}), ("DPMSolverMultistep", {"final_sigmas_type": "zero"}),
         ("DPMSolverMultistep", {"final_sigmas_type": "sigma_min"}), ("PNDM", {})]
IDS = ["ddim", "dpm_zero", "dpm_sigma_min", "pndm"]
VPRED = {"prediction_type": "v_prediction"}


def test_unet_sd21_768_vs_reference_golden(cuda_lib):
    """SD-2.1 768-v: bs=2, 96x96 latents, t=981, against the unmodified reference UNet run on the CPU."""
    from b200sd.model import UNetModel

    gold = np.load(os.path.join(GOLD, "unet_sd21_768.npz"))
    cfg = config.SD21_UNET
    sd = config.random_state_dict(config.unet_param_shapes(cfg), seed=int(gold["weight_seed"]))
    g = torch.Generator().manual_seed(int(gold["input_seed"]))
    x = torch.randn(2, 4, 96, 96, generator=g)
    c = torch.randn(2, 1024, 1, 77, generator=g)
    m = UNetModel(cfg, sd, batch=2, height=96, width=96, use_cuda_graph=True)
    del sd
    t = np.array([float(gold["timestep"])] * 2, np.float16)
    out = m(sample=x.half().numpy(), timestep=t, encoder_hidden_states=c.half().numpy())["noise_pred"]
    _check(out, gold["noise_pred_ORIGINAL"], "SD-2.1 768-v unet vs reference golden")


def test_unet_sd21_768_launches_match_fp64_reference(cuda_lib, monkeypatch):
    """Every GEMM / convolution launch of one eager SD-2.1 forward at batch 2, 96x96 (M = 18432 rows at level 0), with
    the plan the tile planner picks, against the reference of that launch on the live activations."""
    from b200sd.model import UNetModel

    lib = cuda_lib
    for k in ("B200SD_CLUSTER_SPLITK", "B200SD_STAGED", "B200SD_FUSED", "B200SD_HALO_TMA"):
        monkeypatch.delenv(k, raising=False)
    sd = config.random_state_dict(config.unet_param_shapes(config.SD21_UNET), seed=5, dtype=torch.float16)
    m = UNetModel(config.SD21_UNET, sd, batch=2, height=96, width=96, use_cuda_graph=False)
    rep = _Replay(lib, "sd21_768_b2")
    monkeypatch.setattr(lib, "linear", rep.linear)
    monkeypatch.setattr(lib, "conv3x3", rep.conv3x3)
    m(**_model_inputs(m, seed=9))
    torch.cuda.synchronize()
    print("\n" + rep.report())
    assert any(key[1] == 2 * 96 * 96 for key in rep.plans), "no launch over the 18432 level-0 rows was seen"


def test_attention_level0_self_attention_9216_tokens(cuda_lib, monkeypatch):
    """Level-0 self-attention of the 768-v UNet: 5 heads of 64 over 96 * 96 = 9216 tokens, batch 2 (720 query tiles),
    with the schedule the cost model picks and with one CTA per query tile."""
    from test_ops_gpu import _attn_ref, _close, _rand

    batch, heads, s = 2, 5, 9216
    q, k, v = _rand(batch * s, heads * 64, seed=1), _rand(batch * s, heads * 64, seed=2), _rand(batch * s, heads * 64, seed=3)
    ref = _attn_ref(q, k, v, batch, heads, s, s)
    out = cuda_lib.attention(q, k, v, batch, heads, s, s)
    _close(out, ref, 3e-3, 3e-3, "attention 2x5x9216x9216 (default schedule)")
    assert torch.equal(out, cuda_lib.attention(q, k, v, batch, heads, s, s))
    assert int(cuda_lib._attention_workspace(q.device)[:65536].max()) == 0
    monkeypatch.setenv("B200SD_ATTN_STREAMK", "0")
    whole = cuda_lib.attention(q, k, v, batch, heads, s, s)
    monkeypatch.delenv("B200SD_ATTN_STREAMK")
    _close(whole, ref, 3e-3, 3e-3, "attention 2x5x9216x9216 (one CTA per query tile)")
    assert (out.float() - whole.float()).abs().max().item() <= 2e-3


def _tiny_pipe(name, kw, **extra):
    from b200sd.pipeline import B200StableDiffusionPipeline
    return B200StableDiffusionPipeline.from_random_init("tiny", images_per_call=2, height=64, width=64, seed=31,
                                                        scheduler=name, scheduler_kwargs=dict(VPRED, **kw), **extra)


@pytest.mark.parametrize("name,kw", CASES, ids=IDS)
def test_vpred_device_loop_vs_oracle(cuda_lib, name, kw):
    """(a) the restated v-prediction sampler replayed on the engine's own model outputs reproduces the recorded latents
    and the final x0 estimate; (b) end to end against the all-oracle loop (the UNet's fp16 error grows by ~2g+1 per step
    under guidance)."""
    pipe = _tiny_pipe(name, kw)
    prompts = ["a red cube", "a blue sphere"]
    steps, g = 5, 5.0
    np.random.seed(5)
    lat0 = np.random.randn(2, 4, 16, 16).astype(np.float16).astype(np.float32)
    emb = pipe._encode_prompt(prompts, True, None)
    rec = []
    den = pipe.denoise(emb, lat0, steps, g, record=rec, return_denoised=True).cpu().clone()
    ref = V.ORACLES[name](steps, **kw)
    assert [r[0] for r in rec] == ref.timesteps
    # (a) scheduler + CFG kernel in isolation
    x = torch.from_numpy(lat0.copy())
    for i, (t, out, lat_dev) in enumerate(rec):
        x, x0 = ref.step(R.cfg_combine(out[:2].cpu(), out[2:].cpu(), g), x)
        assert (lat_dev.cpu() - x).abs().max() < 2e-4 * max(1.0, float(x.abs().max())), (name, kw, i)
    assert (den - x0).abs().max() < 2e-4 * max(1.0, float(x0.abs().max())), (name, kw)
    # (b) end to end
    ucfg = config.TINY_UNET
    usd = config.random_state_dict(config.unet_param_shapes(ucfg), seed=31, dtype=torch.float16)
    ref = V.ORACLES[name](steps, **kw)
    x = torch.from_numpy(lat0.copy())
    embt = torch.from_numpy(emb).float()
    with torch.no_grad():
        for t in ref.timesteps:
            out = R.unet_forward(usd, ucfg, torch.cat([x, x]).half().float(), torch.tensor([float(t)] * 4), embt)
            x, _ = ref.step(R.cfg_combine(out[:2], out[2:], g), x)
    rel = float((rec[-1][2].cpu() - x).abs().max() / x.abs().max())
    print(f"{name} {kw} v-prediction: end-to-end latent rel err after {steps} steps = {rel:.3e}")
    assert rel < 5e-2, (name, kw)


@pytest.mark.parametrize("name,kw", CASES, ids=IDS)
def test_vpred_loop_graph_equals_step_path(cuda_lib, name, kw):
    """(c) the whole-loop CUDA graph against the step-by-step path, bit for bit; the epsilon loop of the same pipeline
    is another graph and another image."""
    pipe = _tiny_pipe(name, kw)
    prompts = ["a red cube", "a blue sphere"]
    np.random.seed(9)
    lat = np.random.randn(2, 4, 16, 16).astype(np.float16)
    run = dict(height=64, width=64, num_inference_steps=6, guidance_scale=5.0, output_type="np", latents=lat)
    a = pipe(prompts, **run).images
    assert pipe.loop_graph and len(pipe._loop_graphs) == 1
    pipe.loop_graph = False
    b = pipe(prompts, **run).images
    pipe.loop_graph = True
    assert np.isfinite(a).all() and np.array_equal(a, b), float(np.abs(a - b).max())
    pipe.scheduler_kwargs["prediction_type"] = "epsilon"
    e = pipe(prompts, **run).images
    assert len(pipe._loop_graphs) == 2 and not np.array_equal(a, e)


@pytest.mark.parametrize("name,kw", CASES, ids=IDS)
def test_vpred_image_to_image_vs_oracle(cuda_lib, name, kw):
    """(d) image-to-image at strength 0.6: encode, noise to timeSteps[startStep] (the same for both prediction types),
    run the remaining v-prediction steps from an empty multistep state, decode -- against the same on the oracle."""
    from b200sd.pipeline import B200StableDiffusionPipeline

    pipe = B200StableDiffusionPipeline.from_random_init("tiny", images_per_call=1, height=64, width=64, seed=31,
                                                        with_vae_encoder=True, scheduler=name,
                                                        scheduler_kwargs=dict(VPRED, **kw))
    img0 = (torch.rand(1, 3, 64, 64, generator=torch.Generator().manual_seed(32)) * 2 - 1).half().numpy()
    steps, g, strength = 8, 6.0, 0.6
    np.random.seed(33)
    out = pipe("a cat", height=64, width=64, num_inference_steps=steps, guidance_scale=g, starting_image=img0,
               strength=strength, output_type="np").images
    np.random.seed(33)
    noise = np.random.randn(1, 4, 16, 16).astype(np.float16).astype(np.float32)
    enc_noise = np.random.randn(1, 4, 16, 16).astype(np.float32)
    ucfg, vcfg = config.TINY_UNET, config.TINY_VAE
    usd = config.random_state_dict(config.unet_param_shapes(ucfg), seed=31, dtype=torch.float16)
    vsd = config.random_state_dict(config.vae_decoder_param_shapes(vcfg), seed=32, dtype=torch.float16)
    esd = config.random_state_dict(config.vae_encoder_param_shapes(vcfg), seed=81, dtype=torch.float16)
    sched = S.make_scheduler(name, steps, **dict(VPRED, **kw))
    start = sched.start_step(strength)
    assert start == 4
    ref = V.ORACLES[name](steps, start=start, **kw)
    emb = torch.from_numpy(pipe._encode_prompt(["a cat"], True, None)).float()
    with torch.no_grad():
        x0 = R.sample_latents(R.vae_encode(esd, vcfg, torch.from_numpy(img0).float()), torch.from_numpy(enc_noise))
        x = torch.from_numpy(sched.add_noise(x0.numpy(), noise, strength))
        for t in ref.timesteps:
            o = R.unet_forward(usd, ucfg, torch.cat([x, x]).half().float(), torch.tensor([float(t)] * 2), emb)
            x, _ = ref.step(R.cfg_combine(o[:1], o[1:], g), x)
        want = R.postprocess_image(R.vae_decode(vsd, vcfg, x / 0.18215)).numpy()
    err = float(np.abs(out - want).max())
    print(f"{name} {kw} v-prediction img2img: image max_abs={err:.3e}")
    assert err < 3e-2


def _sched_cfg(path, **cfg):
    (path / "scheduler" / "scheduler_config.json").write_text(json.dumps(cfg))


def test_from_pretrained_reads_prediction_type(cuda_lib, tmp_path):
    from test_factory_gpu import _model_dir
    from b200sd.pipeline import B200StableDiffusionPipeline as P

    _model_dir(tmp_path, config.TINY_UNET, seed=41)
    emb = torch.randn(2, 96, 1, 77, generator=torch.Generator().manual_seed(3)).half().numpy()
    run = dict(height=64, width=64, num_inference_steps=4, guidance_scale=5.0, output_type="np", seed=4,
               prompt_embeds=emb)
    for override in (None, "DPMSolverMultistep", "PNDM"):
        images = {}
        for pred in ("epsilon", "v_prediction"):
            # the stabilityai/stable-diffusion-2-1 scheduler config (set_alpha_to_one false, steps_offset 1, ...)
            _sched_cfg(tmp_path, _class_name="DDIMScheduler", prediction_type=pred, beta_schedule="scaled_linear",
                       beta_start=0.00085, beta_end=0.012, clip_sample=False, num_train_timesteps=1000,
                       set_alpha_to_one=False, steps_offset=1, skip_prk_steps=True)
            pipe = P.from_pretrained(str(tmp_path), height=64, width=64, scheduler_override=override)
            assert pipe.scheduler_name == (override or "DDIM")
            assert pipe.scheduler_kwargs["prediction_type"] == pred
            images[pred] = pipe("x", **run).images
            key, = pipe._loop_graphs
            assert ("prediction_type", pred) in key[5]
        assert all(np.isfinite(v).all() for v in images.values())
        assert not np.array_equal(images["epsilon"], images["v_prediction"]), override
    _sched_cfg(tmp_path, _class_name="DDIMScheduler", prediction_type="sample")
    with pytest.raises(ValueError, match="prediction_type"):
        P.from_pretrained(str(tmp_path), height=64, width=64)
    _sched_cfg(tmp_path, _class_name="DDIMScheduler", prediction_type="v_prediction")
    with pytest.raises(ValueError, match="prediction_type"):
        P.from_pretrained(str(tmp_path), height=64, width=64, scheduler_override="EulerDiscrete")


def test_from_random_init_sd21_is_a_768_v_pipeline(cuda_lib):
    from b200sd.pipeline import B200StableDiffusionPipeline as P

    with pytest.raises(ValueError, match="v-prediction"):
        P.from_random_init("sd21", scheduler="EulerDiscrete")
    pipe = P.from_random_init("sd21", seed=1)
    assert (pipe.height, pipe.width, pipe.unet.h) == (768, 768, 96)
    assert pipe.scheduler_kwargs == {"prediction_type": "v_prediction"}
    img = pipe("a photo", num_inference_steps=2, guidance_scale=7.5, height=768, width=768, output_type="np",
               seed=3).images
    assert img.shape == (1, 768, 768, 3) and np.isfinite(img).all()
