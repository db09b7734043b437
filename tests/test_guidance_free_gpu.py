"""GPU tests of the guidance-free loop and guidance-embedding (LCM) UNets: the step kernel's guidance-free mode against
its host twin, the guidance-free device loop (loop graph against the step-by-step path, against the same loop run
through the batch-2N UNet on duplicated halves, and the UNet batch it ran at) for SD-2.1-base, SDXL with
Euler-ancestral (trailing), ControlNet and both inpainting kinds, an LCM UNet against the oracle, and every launch of the
batch-1 UNets against its fp64 replay."""
import numpy as np
import pytest
import torch

import model_cases as MC
from b200sd import config
from b200sd import scheduler as S
from b200sd.pipeline import B200StableDiffusionPipeline as P
from b200sd.pipeline import InpaintInputs
from b200sd.rng import NvRandomSource
from b200sd.unet import guidance_scale_embedding
from oracle import restated as R
from test_guidance_free import unet_forward_cond

pytestmark = pytest.mark.gpu

MIN_PSNR = 35.0  # the UNet bar (test_unet_gpu.py)


def _key(value):
    return torch.tensor([np.uint32(value).view(np.int32)], dtype=torch.int32, device="cuda")


@pytest.mark.parametrize("form", ["plain", "noised", "blend", "blend_noised"])
@pytest.mark.parametrize("nhwc", [0, 1])
def test_guidance_free_step_kernel_matches_host(cuda_lib, form, nhwc):
    lib = cuda_lib
    n, c, h, w, c_pad = 2, 4, 16, 24, 8
    g = torch.Generator(device="cuda").manual_seed(3)
    eps = torch.randn(n, c, h, w, device="cuda", generator=g)
    lat = torch.randn(n, c, h, w, device="cuda", generator=g)
    hist = torch.randn(4, n, c, h, w, device="cuda", generator=g)
    st = S.make_scheduler("LMSDiscrete", 20).plan()[5]  # reads and pushes history
    st.noise_scale, st.noise_offset = (0.7, 3) if form.endswith("noised") else (0.0, -1)
    k = P._coeffs(st, 123.0, lib.StepCoeffs())  # the guidance value must not be read
    k.noise_pred_nhwc = nhwc
    x, hh = lat.double().cpu().numpy(), hist.double().cpu().numpy()
    z = None
    if st.noise_offset >= 0:
        src = NvRandomSource(99)
        src.offset = 3
        z = src.normal_array(lat.numel()).reshape(lat.shape)
    e = eps.double().cpu().numpy()
    want, want_x0 = S.apply_plan_host(st, 1.0, e, e, x, hh, z)
    blend = None
    if form.startswith("blend"):
        m = (torch.rand(n, 1, h, w, device="cuda", generator=g) > 0.5).float()
        x0i = torch.randn(n, c, h, w, device="cuda", generator=g)
        zi = torch.randn(n, c, h, w, device="cuda", generator=g)
        blend = (m, x0i, zi, 0.6, 0.8)
        keep = 0.6 * x0i.double().cpu().numpy() + 0.8 * zi.double().cpu().numpy()
        mm = m.double().cpu().numpy()
        want = mm * want + (1 - mm) * keep
    npred = eps.permute(0, 2, 3, 1).contiguous() if nhwc else eps
    unet_in = torch.full((2 * n, h, w, c_pad), 7.0, dtype=torch.float16, device="cuda")
    den = torch.zeros_like(lat)
    lib.scheduler_step_guidance_free(npred, lat, k, st.noise_scale, _key(99) if z is not None else None, 3,
                                     blend=blend, hist=hist, denoised=den, unet_in=unet_in)
    np.testing.assert_allclose(lat.cpu().numpy(), want, rtol=1e-5, atol=1e-5)
    np.testing.assert_allclose(den.cpu().numpy(), want_x0, rtol=1e-5, atol=1e-5)
    np.testing.assert_allclose(hist.cpu().numpy(), hh, rtol=1e-6, atol=1e-6)
    assert torch.equal(unet_in[:n, :, :, :c], lat.permute(0, 2, 3, 1).half())
    assert (unet_in[n:] == 7.0).all() and (unet_in[:n, :, :, c:] == 7.0).all()  # one half, channels [0, c) only
    with pytest.raises(lib.B200SDError, match="one prediction per image"):
        lib.scheduler_step_guidance_free(torch.zeros(2 * n, c, h, w, device="cuda"), lat, k)


def _run_three_ways(pipe, emb, lat, steps, g, **kw):
    """-> (loop graph, step-by-step, batch-2N guided loop at guidance 1 on duplicated halves) final latents, and the
    rows of every time table the guidance-free loop built."""
    rows = []
    tt = type(pipe.unet).time_table

    def table(self, ts_rows, r=None):
        out = tt(self, ts_rows, r)
        rows.append(out.shape[1])
        return out
    pipe.unet.time_table = table.__get__(pipe.unet)
    try:
        graph = pipe.denoise(emb, lat, steps, g, **kw).clone()
    finally:
        del pipe.unet.time_table
    step = pipe.denoise(emb, lat, steps, g, record=[], **kw).clone()
    pipe.do_classifier_free_guidance = lambda _g: True
    try:
        dup = pipe.denoise(emb, lat, steps, 1.0, record=[], **kw).clone()
    finally:
        del pipe.do_classifier_free_guidance
    return graph, step, dup, rows


def _check(what, pipe, emb, lat, steps, g, **kw):
    graph, step, dup, rows = _run_three_ways(pipe, emb, lat, steps, g, **kw)
    assert torch.equal(graph, step), f"{what}: loop graph != step-by-step path"
    psnr = R.compute_psnr(graph.cpu().double(), dup.cpu().double())
    print(f"{what}: guidance-free vs batch-2N max_abs={float((graph - dup).abs().max()):.3e} psnr={psnr:.1f} dB")
    assert psnr >= MIN_PSNR, f"{what}: psnr {psnr:.1f}"
    assert rows and set(rows) == {pipe.images_per_call}, f"{what}: UNet time-table rows {rows}"


@pytest.mark.parametrize("n", [1, 2])
def test_sd21_base_txt2img_guidance_free(cuda_lib, n):
    pipe = P.from_random_init("sd21-base", images_per_call=n, seed=1)
    prompts = ["a cat", "a dog"][:n]
    emb = pipe._encode_prompt(prompts, False, None)
    assert emb.shape[0] == 2 * n
    lat = np.random.RandomState(2).standard_normal((n, 4, 64, 64)).astype(np.float32)
    _check(f"sd21-base n={n}", pipe, emb, lat, 6, 1.0)
    half = pipe.denoise(emb[n:], lat, 6, 0.0).clone()  # N rows or the 2N uncond-first layout: the same loop
    assert torch.equal(half, pipe.denoise(emb, lat, 6, 1.0))
    out = pipe(prompts[0] if n == 1 else prompts, num_inference_steps=2, guidance_scale=1.0, seed=5, output_type="np")
    assert np.isfinite(out.images).all()


@pytest.mark.parametrize("steps", [1, 4])
def test_sdxl_512_euler_ancestral_trailing(cuda_lib, steps):
    pipe = P.from_random_init("sdxl-base", seed=1, scheduler="EulerAncestralDiscrete",
                              scheduler_kwargs={"timestep_spacing": "trailing"})
    g = torch.Generator().manual_seed(3)
    emb = (torch.randn(1, 2048, 1, 77, generator=g) * 0.5).half().repeat(2, 1, 1, 1)
    pooled = torch.randn(1, 1280, generator=g).repeat(2, 1)
    tid = torch.tensor([[512.0, 512.0, 0.0, 0.0, 512.0, 512.0]] * 2)
    sched = S.make_scheduler("EulerAncestralDiscrete", steps, timestep_spacing="trailing")
    lat = (torch.randn(1, 4, 64, 64, generator=g) * sched.init_noise_sigma).numpy()
    _check(f"sdxl-512 euler-a {steps}", pipe, emb, lat, steps, 0.0, time_ids=tid, text_embeds=pooled, noise_key=11)


def test_controlnet_guidance_free(cuda_lib):
    pipe = P.from_random_init("sd21-base", seed=1, controlnet_cfgs=[config.SD21_CONTROLNET])
    emb = pipe._encode_prompt(["a house"], False, None)
    cond = np.random.RandomState(4).rand(3, 512, 512).astype(np.float32)
    cc = pipe.prepare_control_cond([cond], False, 1, 1)
    lat = np.random.RandomState(5).standard_normal((1, 4, 64, 64)).astype(np.float32)
    _check("controlnet sd21", pipe, emb, lat, 4, 1.0, controlnet_cond=cc)


@pytest.mark.parametrize("cin", [4, 9])
def test_inpainting_guidance_free(cuda_lib, cin):
    pipe = P.from_random_init("sd21-base", seed=1, unet_cfg=dict(config.SD21_BASE_UNET, in_channels=cin))
    emb = pipe._encode_prompt(["a vase"], False, None)
    rs = np.random.RandomState(6)
    mask = np.zeros((1, 1, 64, 64), np.float32)
    mask[..., :, 20:] = 1.0
    noise = rs.standard_normal((1, 4, 64, 64)).astype(np.float32)
    inp = InpaintInputs(mask, rs.standard_normal((1, 4, 64, 64)).astype(np.float32), noise,
                        rs.standard_normal((1, 4, 64, 64)).astype(np.float32))
    _check(f"inpaint cin={cin}", pipe, emb, noise, 4, 1.0, inpaint=inp)


def test_lcm_unet_forward_matches_oracle(cuda_lib):
    from b200sd.model import UNetModel
    cfg = dict(config.SD15_UNET, time_cond_proj_dim=256)
    sd = config.random_state_dict(config.unet_param_shapes(cfg), seed=7, dtype=torch.float16)
    m = UNetModel(cfg, sd, batch=2, height=64, width=64)
    g = torch.Generator().manual_seed(8)
    x = torch.randn(2, 4, 64, 64, generator=g).half().float()
    ctx = torch.randn(2, 768, 1, 77, generator=g).half().float()
    t = torch.tensor([759.0, 259.0])  # two rows with their own timestep and condition
    cond = torch.cat([guidance_scale_embedding(8.0, 256), guidance_scale_embedding(3.0, 256)])
    out = m.forward_device(x.cuda(), t.cuda(), ctx.half().cuda(), timestep_cond=cond.cuda()).cpu()
    with torch.no_grad():
        ref = unet_forward_cond({k: v.float() for k, v in sd.items()}, cfg, x, t, ctx, cond)
    err = float((out - ref).abs().max())
    psnr = R.compute_psnr(out, ref)
    print(f"lcm sd15 forward: max_abs={err:.3e} psnr={psnr:.1f} dB")
    assert err <= 1e-2 and psnr >= MIN_PSNR
    plain = m.forward_device(x.cuda(), t.cuda(), ctx.half().cuda(),
                             timestep_cond=guidance_scale_embedding(1.0, 256, 2).cuda()).cpu()
    assert not torch.allclose(plain, out, atol=1e-3)  # the condition reaches the UNet
    with pytest.raises(ValueError, match="timestep_cond"):
        m.forward_device(x.cuda(), t.cuda(), ctx.half().cuda())


def test_lcm_pipeline_reproducible_and_graph_equals_step(cuda_lib):
    pipe = P.from_random_init("sd15", seed=1, scheduler="LCM",
                              unet_cfg=dict(config.SD15_UNET, time_cond_proj_dim=256))
    assert not pipe.do_classifier_free_guidance(8.0)
    a = pipe("a cat", num_inference_steps=4, guidance_scale=8.0, seed=42, output_type="np").images
    b = pipe("a cat", num_inference_steps=4, guidance_scale=8.0, seed=42, output_type="np").images
    assert np.array_equal(a, b) and np.isfinite(a).all()
    emb = pipe._encode_prompt(["a cat"], False, None)
    lat = np.random.RandomState(9).standard_normal((1, 4, 64, 64)).astype(np.float32)
    graph = pipe.denoise(emb, lat, 4, 8.0, noise_key=42).clone()
    step = pipe.denoise(emb, lat, 4, 8.0, noise_key=42, record=[]).clone()
    assert torch.equal(graph, step)
    assert not torch.equal(graph, pipe.denoise(emb, lat, 4, 2.0, noise_key=42))  # guidance enters as an embedding


BATCH1 = {"sd21_b1": ("sd21_b2", config.SD21_BASE_UNET), "sd15_b1": ("sd15_b2", config.SD15_UNET),
          "sdxl_512_b1": ("sdxl_512x512_b2", config.SDXL_BASE_UNET),
          "sdxl_1024_b1": ("sdxl_1024_b2", config.SDXL_BASE_UNET), "controlnet_sd21_b1": ("controlnet_sd21", None)}


def _build_b1(name):
    from b200sd.controlnet import ControlNetModel
    from b200sd.model import UNetModel
    shipped, cfg = BATCH1[name]
    h, w = MC.latent_hw(shipped)
    if cfg is None:
        ccfg = config.SD21_CONTROLNET
        sd = config.random_state_dict(config.controlnet_param_shapes(ccfg), seed=5, dtype=torch.float16)
        return ControlNetModel(ccfg, sd, batch=1, height=h, width=w, use_cuda_graph=False)
    sd = config.random_state_dict(config.unet_param_shapes(cfg), seed=5, dtype=torch.float16)
    return UNetModel(cfg, sd, batch=1, height=h, width=w, use_cuda_graph=False)


@pytest.mark.parametrize("name", list(BATCH1))
def test_batch1_gemm_launches_match_fp64(cuda_lib, monkeypatch, name):
    """The guidance-free loop runs the UNets and ControlNets at batch N = 1: an odd M no shipped launch has had."""
    from test_gemm_plans_gpu import _Replay
    lib = cuda_lib
    for k in ("B200SD_CLUSTER_SPLITK", "B200SD_STAGED", "B200SD_FUSED", "B200SD_HALO_TMA"):
        monkeypatch.delenv(k, raising=False)
    m = _build_b1(name)
    rep = _Replay(lib, name)
    monkeypatch.setattr(lib, "linear", rep.linear)
    monkeypatch.setattr(lib, "conv3x3", rep.conv3x3)
    m(**MC.model_inputs(m, seed=9))
    torch.cuda.synchronize()
    print(f"\n{rep.report()}")
    assert rep.plans


@pytest.mark.parametrize("name", list(BATCH1))
def test_batch1_op_launches_match_fp64(cuda_lib, monkeypatch, name):
    from test_op_launches_gpu import _Replay
    lib = cuda_lib
    for k in ("B200SD_CLUSTER_SPLITK", "B200SD_STAGED", "B200SD_FUSED", "B200SD_HALO_TMA"):
        monkeypatch.delenv(k, raising=False)
    m = _build_b1(name)
    rep = _Replay(lib, name)
    rep.install(monkeypatch)
    m(**MC.model_inputs(m, seed=9))
    torch.cuda.synchronize()
    print(f"\n{rep.report()}")
    assert {"attention", "group_norm", "linear_small", "timestep_embedding"} <= {key[0] for key in rep.rows}


def test_from_pretrained_lcm_directory(cuda_lib, tmp_path):
    import json

    from test_factory_gpu import _model_dir, _write_component
    ucfg = dict(config.TINY_UNET, time_cond_proj_dim=32)
    usd, _ = _model_dir(tmp_path, ucfg, seed=21)
    lcm_cfg = {"_class_name": "LCMScheduler", "original_inference_steps": 50, "timestep_scaling": 10.0,
               "clip_sample": False, "beta_schedule": "scaled_linear", "prediction_type": "epsilon"}
    (tmp_path / "scheduler" / "scheduler_config.json").write_text(json.dumps(lcm_cfg))
    pipe = P.from_pretrained(str(tmp_path), height=64, width=64)
    assert pipe.scheduler_name == "LCM" and pipe.unet.engine.time_cond_dim == 32
    img = pipe("a cat", height=64, width=64, num_inference_steps=4, guidance_scale=8.0, seed=3, output_type="np").images
    assert img.shape == (1, 64, 64, 3) and np.isfinite(img).all()
    del usd["time_embedding.cond_proj.weight"]
    _write_component(tmp_path, "unet", usd, ucfg, "UNet2DConditionModel")
    with pytest.raises(KeyError):
        P.from_pretrained(str(tmp_path), height=64, width=64)


def test_from_pretrained_turbo_directory(cuda_lib, tmp_path):
    import json

    from test_factory_gpu import _model_dir
    _model_dir(tmp_path, config.TINY_UNET, seed=22)
    turbo = {"_class_name": "EulerAncestralDiscreteScheduler", "timestep_spacing": "trailing", "steps_offset": 1,
             "beta_schedule": "scaled_linear", "prediction_type": "epsilon", "interpolation_type": "linear",
             "use_karras_sigmas": False}
    (tmp_path / "scheduler" / "scheduler_config.json").write_text(json.dumps(turbo))
    pipe = P.from_pretrained(str(tmp_path), height=64, width=64)
    assert pipe.scheduler_name == "EulerAncestralDiscrete" and pipe.scheduler_kwargs["timestep_spacing"] == "trailing"
    img = pipe("a cat", height=64, width=64, num_inference_steps=1, guidance_scale=0.0, seed=3, output_type="np").images
    assert img.shape == (1, 64, 64, 3) and np.isfinite(img).all()
