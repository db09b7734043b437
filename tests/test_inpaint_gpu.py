"""GPU tests of inpainting: the SD-1.5 9-channel UNet against the unmodified reference (tests/golden/make_golden_inpaint.py)
and every GEMM / convolution launch of it against an fp64 reference of that launch; the step kernel's blend against
float64; the inpainting device loop (4-channel blend and 9-channel UNet, all six schedulers) against the diffusers
restatement (tests/inpaint_oracle.py); loop graph against step path; ``from_pretrained``; the C handle at 9 channels."""
import json
import os

import numpy as np
import pytest
import torch

import inpaint_oracle as O
from b200sd import config
from b200sd import scheduler as S
from b200sd.rng import NvRandomSource
from oracle import restated as R
from model_cases import model_inputs as _model_inputs
from test_gemm_plans_gpu import _Replay
from test_unet_gpu import _check

pytestmark = pytest.mark.gpu
GOLD = os.path.join(os.path.dirname(__file__), "golden")
ALL = ["DDIM", "DPMSolverMultistep", "PNDM", "EulerDiscrete", "EulerAncestralDiscrete", "LMSDiscrete"]
TINY9 = dict(config.TINY_UNET, in_channels=9)


def test_unet_sd15_inpaint_vs_reference_golden(cuda_lib):
    """SD-1.5 with in_channels = 9 (conv_in over 16 padded input channels): bs=2, 64x64 latents."""
    from b200sd.model import UNetModel

    gold = np.load(os.path.join(GOLD, "unet_sd15_inpaint.npz"))
    cfg = dict(config.SD15_UNET, in_channels=9)
    sd = config.random_state_dict(config.unet_param_shapes(cfg), seed=int(gold["weight_seed"]))
    g = torch.Generator().manual_seed(int(gold["input_seed"]))
    x = torch.randn(2, 9, 64, 64, generator=g)
    c = torch.randn(2, 768, 1, 77, generator=g)
    m = UNetModel(cfg, sd, batch=2, height=64, width=64)
    assert m.engine.in_pad == 16
    del sd
    t = np.array([float(gold["timestep"])] * 2, np.float16)
    out = m(sample=x.half().numpy(), timestep=t, encoder_hidden_states=c.half().numpy())["noise_pred"]
    _check(out, gold["noise_pred_ORIGINAL"], "SD-1.5 inpainting unet vs reference golden")


def test_unet_sd15_inpaint_launches_match_fp64_reference(cuda_lib, monkeypatch):
    from b200sd.model import UNetModel

    lib = cuda_lib
    for k in ("B200SD_CLUSTER_SPLITK", "B200SD_STAGED", "B200SD_FUSED", "B200SD_HALO_TMA"):
        monkeypatch.delenv(k, raising=False)
    cfg = dict(config.SD15_UNET, in_channels=9)
    sd = config.random_state_dict(config.unet_param_shapes(cfg), seed=5, dtype=torch.float16)
    m = UNetModel(cfg, sd, batch=2, height=64, width=64, use_cuda_graph=False)
    rep = _Replay(lib, "sd15_inpaint_b2")
    monkeypatch.setattr(lib, "linear", rep.linear)
    monkeypatch.setattr(lib, "conv3x3", rep.conv3x3)
    m(**_model_inputs(m, seed=9))
    torch.cuda.synchronize()
    print("\n" + rep.report())
    assert any(key[0] == "conv3x3" and key[3] == 9 * 16 for key in rep.plans), "conv_in at Ci = 16 was not seen"


# ---------------------------------------------------------------- blend kernel
def _step_args(n, c, hw, seed):
    g = torch.Generator(device="cuda").manual_seed(seed)
    h, w = hw
    r = lambda *s: torch.randn(*s, generator=g, device="cuda")  # noqa: E731
    return dict(eps=r(2 * n, c, h, w), lat=r(n, c, h, w), hist=r(4, n, c, h, w), x0=r(n, c, h, w), z=r(n, c, h, w))


def _coeffs(lib):
    k = lib.StepCoeffs()
    k.guidance, k.cx, k.ce, k.x0_cx, k.x0_ce = 5.0, 0.9, -0.3, 1.2, -0.7
    k.ch[1], k.x0_ch[1], k.n_hist = 0.25, -0.5, 2
    k.push_eps_slot, k.push_x_slot, k.push_x0_slot = 0, 2, 3
    return k


@pytest.mark.parametrize("n,hw", [(1, (7, 9)), (2, (5, 13)), (2, (16, 16))])
@pytest.mark.parametrize("noised", [False, True])
def test_blend_kernel_vs_fp64(cuda_lib, n, hw, noised):
    lib = cuda_lib
    c, c_pad = 4, 16
    t = _step_args(n, c, hw, seed=n * 100 + hw[0])
    key = torch.tensor([1234], dtype=torch.int32, device="cuda")
    kw = dict(noise_scale=0.7, key=key, offset=3) if noised else {}
    k = _coeffs(lib)
    mask = (torch.rand(n, 1, *hw, generator=torch.Generator(device="cuda").manual_seed(7), device="cuda") > 0.5).float()
    a, b = 0.8, 0.6

    def run(m, a_, b_, blend=True):
        lat, hist, den = t["lat"].clone(), t["hist"].clone(), torch.zeros_like(t["lat"])
        unet_in = torch.full((2 * n, *hw, c_pad), 7.0, dtype=torch.float16, device="cuda")
        if blend:
            lib.cfg_scheduler_step_blend(t["eps"], lat, k, m, t["x0"], t["z"], a_, b_, hist=hist, denoised=den,
                                         unet_in=unet_in, **kw)
        elif noised:
            lib.cfg_scheduler_step_noised(t["eps"], lat, k, 0.7, key, 3, hist=hist, denoised=den, unet_in=unet_in)
        else:
            lib.cfg_scheduler_step(t["eps"], lat, k, hist=hist, denoised=den, unet_in=unet_in)
        return lat, hist, den, unet_in

    lat, hist, den, unet_in = run(mask, a, b)
    # float64 reference
    d = {k_: v.double() for k_, v in t.items()}
    e = d["eps"][:n] + 5.0 * (d["eps"][n:] - d["eps"][:n])
    xp = 0.9 * d["lat"] - 0.3 * e + 0.25 * d["hist"][1]
    x0 = 1.2 * d["lat"] - 0.7 * e - 0.5 * d["hist"][1]
    if noised:
        src = NvRandomSource(1234)
        src.offset = 3
        xp = xp + 0.7 * torch.from_numpy(src.normal_array(n * c * hw[0] * hw[1])).reshape(xp.shape).double().cuda()
    m = mask.double()
    ref = m * xp + (1 - m) * (a * d["x0"] + b * d["z"])
    assert (lat.double() - ref).abs().max() < 1e-5 * max(1.0, float(ref.abs().max()))
    assert (den.double() - x0).abs().max() < 1e-5 * max(1.0, float(x0.abs().max()))  # pre-blend
    assert (hist[0].double() - e).abs().max() < 1e-5 * float(e.abs().max())  # history pushes: pre-blend
    assert torch.equal(hist[2], t["lat"]) and torch.equal(hist[3], den)
    nhwc = lat.permute(0, 2, 3, 1).half()
    assert torch.equal(unet_in[:n, ..., :c], nhwc) and torch.equal(unet_in[n:, ..., :c], nhwc)
    assert bool((unet_in[..., c:] == 7.0).all()), "channels [c, c_pad) were written"
    # m = 1: bit-identical to the plain / noised step; m = 0, b = 0: the image latents exactly
    ones = run(torch.ones_like(mask), a, b)
    plain = run(None, 0, 0, blend=False)
    for u, v in zip(ones, plain):
        assert torch.equal(u, v)
    zeros = run(torch.zeros_like(mask), 1.0, 0.0)
    assert torch.equal(zeros[0], t["x0"]) and torch.equal(zeros[2], plain[2])


# ---------------------------------------------------------------- device loop
def _pipe(name, cin, images=2, px=(64, 64), **kw):
    from b200sd.pipeline import B200StableDiffusionPipeline
    ucfg = TINY9 if cin == 9 else config.TINY_UNET
    return B200StableDiffusionPipeline.from_random_init("tiny", images_per_call=images, height=px[0], width=px[1],
                                                        seed=31, scheduler=name, with_vae_encoder=True, unet_cfg=ucfg,
                                                        **kw)


def _images(seed, b=2, px=(64, 64)):
    """Images and masks: discs at 64^2; at any other size the left third of the image (a mask that changes when h and
    w are swapped)."""
    g = torch.Generator().manual_seed(seed)
    img = (torch.rand(b, 3, *px, generator=g) * 2 - 1).half().numpy()
    yy, xx = np.meshgrid(np.arange(px[0]), np.arange(px[1]), indexing="ij")
    if px == (64, 64):
        mask = np.stack([((yy - 20 - 8 * i) ** 2 + (xx - 30) ** 2 < 300).astype(np.float32)[None] for i in range(b)])
    else:
        mask = np.stack([(xx < px[1] // 3).astype(np.float32)[None] for _ in range(b)])
    return img, mask


def _loop_cases():
    out = [(name, cin, 1.0, {}) for cin in (4, 9) for name in ALL]
    out += [(name, cin, 0.6, {}) for cin in (4, 9) for name in ("DDIM", "DPMSolverMultistep")]
    out += [("DPMSolverMultistep", 9, 1.0, {"prediction_type": "v_prediction"}),
            ("DDIM", 4, 0.6, {"prediction_type": "v_prediction"})]
    return out


@pytest.mark.parametrize("name,cin,strength,skw", _loop_cases(),
                         ids=lambda v: v if isinstance(v, str) else (f"s{v}" if isinstance(v, float) else
                                                                      (f"c{v}" if isinstance(v, int) else
                                                                       ("vpred" if v else "eps"))))
def test_inpaint_device_loop_vs_oracle(cuda_lib, name, cin, strength, skw):
    _inpaint_device_loop_vs_oracle(name, cin, strength, skw)


@pytest.mark.parametrize("cin", [4, 9])
def test_inpaint_device_loop_vs_oracle_non_square(cuda_lib, cin):
    """DDIM at 64x96 pixels (16x24 latents) with the left third masked."""
    _inpaint_device_loop_vs_oracle("DDIM", cin, 1.0, {}, px=(64, 96))


def _inpaint_device_loop_vs_oracle(name, cin, strength, skw, px=(64, 64)):
    """(a) the restated inpaint loop fed the engine's recorded noise predictions reproduces the recorded latents;
    (b) ``__call__`` end to end against the all-oracle pipeline (restated UNet and VAE); (c) 4-channel UNets: the
    latents where the latent mask is 0 are the image latents bit for bit."""
    from b200sd.pipeline import InpaintInputs, latent_mask, prepare_mask_and_masked_image

    pipe = _pipe(name, cin, px=px, scheduler_kwargs=skw)
    steps, g, key = 6, 5.0, 77
    img, mask = _images(3, px=px)
    lh, lw = px[0] // 4, px[1] // 4  # the tiny VAE downsamples by 4
    emb = pipe._encode_prompt(["a red cube", "a blue sphere"], True, None)
    gen = torch.Generator().manual_seed(4)
    noise = torch.randn(2, 4, lh, lw, generator=gen).half().float()
    x0_img = torch.randn(2, 4, lh, lw, generator=gen)
    masked_lat = torch.randn(2, 4, lh, lw, generator=gen)
    sched = S.make_scheduler(name, steps, **pipe.scheduler_kwargs)
    start = sched.inpaint_start_step(strength)
    m_img, _ = prepare_mask_and_masked_image(img, mask)
    m_lat = latent_mask(m_img, pipe.vae_scale_factor)
    assert m_lat.shape[-2:] == (lh, lw)
    if start:
        a, b = sched.noise_coeffs(start)
        lat0 = (np.float32(a) * x0_img.numpy() + np.float32(b) * noise.numpy()).astype(np.float32)
    else:
        lat0 = (noise * sched.init_noise_sigma).numpy()
    inp = InpaintInputs(m_lat, x0_img.numpy(), noise.numpy(), masked_lat.numpy())
    rec = []
    final = pipe.denoise(emb, lat0, steps, g, record=rec, start_step=start, noise_key=key, inpaint=inp).cpu().clone()
    src = NvRandomSource(key)

    def step_noise(i):
        src.offset = i
        return torch.from_numpy(src.normal_array(noise.numel()).reshape(noise.shape))

    calls = []
    encode = lambda im: (calls.append(1), x0_img if len(calls) == 1 and (cin == 4 or start) else masked_lat)[1]  # noqa
    want = []
    O.inpaint(None, encode, img, mask, noise, name, steps, g, strength=strength, in_channels=cin,
              step_noise=step_noise, model_outputs=[r[1].cpu() for r in rec], record=want, **skw,
              **({"final_sigmas_type": "zero"} if name == "DPMSolverMultistep" else {}))
    assert len(want) == len(rec)
    for i, (w, (_, _, got)) in enumerate(zip(want, rec)):
        assert (got.cpu().double() - w).abs().max() < 2e-4 * max(1.0, float(w.abs().max())), (name, cin, i)
    assert torch.equal(final, rec[-1][2].cpu())
    if cin == 4:
        keep = torch.from_numpy(m_lat).expand_as(final) == 0
        assert torch.equal(final[keep], x0_img[keep])
    # (b) end to end through __call__, against the restated UNet / VAE
    np.random.seed(8)
    out = pipe(["a red cube", "a blue sphere"], height=px[0], width=px[1], num_inference_steps=steps, guidance_scale=g,
               starting_image=img, mask_image=mask, strength=strength, output_type="np", seed=key, rng="nvidia").images
    assert out.shape == (2, *px, 3)
    ucfg = TINY9 if cin == 9 else config.TINY_UNET
    vcfg = config.TINY_VAE
    usd = config.random_state_dict(config.unet_param_shapes(ucfg), seed=31, dtype=torch.float16)
    vsd = config.random_state_dict(config.vae_decoder_param_shapes(vcfg), seed=32, dtype=torch.float16)
    esd = config.random_state_dict(config.vae_encoder_param_shapes(vcfg), seed=81, dtype=torch.float16)
    src0 = NvRandomSource(key)
    lat_noise = torch.from_numpy(np.stack([src0.normal_array(4 * lh * lw).reshape(4, lh, lw)
                                           for _ in range(2)])).float()
    np.random.seed(8)
    enc_noises = []

    def encode_ref(im):
        z = torch.from_numpy(np.random.randn(2, 4, lh, lw).astype(np.float32))
        enc_noises.append(z)
        return R.sample_latents(R.vae_encode(esd, vcfg, im.half().float()), z)

    def unet_ref(x, t):
        return R.unet_forward(usd, ucfg, x.float().half().float(), torch.tensor([float(np.float16(t))] * 4),
                              torch.from_numpy(emb).float()).double()

    src_off = 2  # the nvidia source continues after the latents' two draws

    def step_noise_ref(i):
        s = NvRandomSource(key)
        s.offset = src_off + i
        return torch.from_numpy(s.normal_array(noise.numel()).reshape(noise.shape))
    with torch.no_grad():
        x = O.inpaint(unet_ref, encode_ref, torch.from_numpy(img).float(), mask, lat_noise, name, steps, g,
                      strength=strength, in_channels=cin, step_noise=step_noise_ref, **skw,
                      **({"final_sigmas_type": "zero"} if name == "DPMSolverMultistep" else {}))
        ref_img = R.postprocess_image(R.vae_decode(vsd, vcfg, x.float() / 0.18215)).numpy()
    err = float(np.abs(out - ref_img).max())
    print(f"inpaint {name} c{cin} strength {strength} {skw} {px[0]}x{px[1]}: image max_abs={err:.3e}")
    assert err < 5e-2, err


@pytest.mark.parametrize("cin", [4, 9])
def test_inpaint_loop_graph_equals_step_path(cuda_lib, cin):
    """One captured loop graph serves two masks and images; bit-identical to the step path; the 9-channel
    conditioning in UNet input channels 4..8 survives every step."""
    pipe = _pipe("DPMSolverMultistep", cin)
    run = dict(height=64, width=64, num_inference_steps=5, guidance_scale=5.0, output_type="np", seed=3)
    outs = []
    for seed in (3, 4):
        img, mask = _images(seed)
        mask = mask[:, :, ::-1].copy() if seed == 4 else mask
        np.random.seed(seed)
        a = pipe(["a", "b"], starting_image=img, mask_image=mask, **run).images
        assert len(pipe._loop_graphs) == 1 and pipe._loop_graphs and list(pipe._loop_graphs)[0][-1] == (
            "unet9" if cin == 9 else "blend")
        if cin == 9:
            cond = pipe._inpaint_bufs["unet_in"][:, 4:].permute(0, 2, 3, 1).half()
            x_in = pipe.unet._x_nhwc
            assert torch.equal(x_in[:2, ..., 4:9], cond) and torch.equal(x_in[2:, ..., 4:9], cond)
        pipe.loop_graph = False
        np.random.seed(seed)
        b = pipe(["a", "b"], starting_image=img, mask_image=mask, **run).images
        pipe.loop_graph = True
        assert np.isfinite(a).all() and np.array_equal(a, b), float(np.abs(a - b).max())
        outs.append(a)
    assert not np.array_equal(outs[0], outs[1])
    if cin == 4:  # text-to-image on the same pipeline is another graph
        pipe(["a", "b"], **run)
        assert len(pipe._loop_graphs) == 2


def _write_dir(path, ucfg, seed):
    from test_factory_gpu import _write_component
    usd = config.random_state_dict(config.unet_param_shapes(ucfg), seed=seed, dtype=torch.float16)
    vcfg = config.TINY_VAE
    vsd = config.random_state_dict(config.vae_decoder_param_shapes(vcfg), seed=seed + 1, dtype=torch.float16)
    vsd.update(config.random_state_dict(config.vae_encoder_param_shapes(vcfg), seed=seed + 2, dtype=torch.float16))
    _write_component(path, "unet", usd, ucfg, "UNet2DConditionModel")
    _write_component(path, "vae", vsd, vcfg, "AutoencoderKL")
    os.makedirs(path / "scheduler", exist_ok=True)
    (path / "scheduler" / "scheduler_config.json").write_text(json.dumps({"_class_name": "DDIMScheduler"}))
    return usd, vsd


@pytest.mark.parametrize("cin", [4, 9])
def test_from_pretrained_inpainting(cuda_lib, tmp_path, cin):
    from b200sd.pipeline import B200StableDiffusionPipeline as P

    ucfg = TINY9 if cin == 9 else config.TINY_UNET
    usd, vsd = _write_dir(tmp_path, ucfg, seed=71)
    pipe = P.from_pretrained(str(tmp_path), height=64, width=64, with_vae_encoder=True)
    assert pipe.unet.in_channels == cin and pipe.latent_channels == 4 and pipe._latents.shape[1] == 4
    img, mask = _images(5, b=1)
    emb = torch.randn(2, 96, 1, 77, generator=torch.Generator().manual_seed(3)).half().numpy()
    steps, g = 5, 6.0
    np.random.seed(2)
    out = pipe("x", height=64, width=64, num_inference_steps=steps, guidance_scale=g, starting_image=img,
               mask_image=mask[0, 0], output_type="np", prompt_embeds=emb).images
    vcfg = config.TINY_VAE
    np.random.seed(2)
    lat_noise = torch.from_numpy(np.random.randn(1, 4, 16, 16).astype(np.float16).astype(np.float32))

    def encode_ref(im):
        z = torch.from_numpy(np.random.randn(1, 4, 16, 16).astype(np.float32))
        return R.sample_latents(R.vae_encode(vsd, vcfg, im.half().float()), z)

    def unet_ref(x, t):
        return R.unet_forward(usd, ucfg, x.float().half().float(), torch.tensor([float(t)] * 2),
                              torch.from_numpy(emb).float()).double()
    with torch.no_grad():
        x = O.inpaint(unet_ref, encode_ref, torch.from_numpy(img).float(), mask[0, 0], lat_noise, "DDIM", steps, g,
                      in_channels=cin)
        ref_img = R.postprocess_image(R.vae_decode(vsd, vcfg, x.float() / 0.18215)).numpy()
    err = float(np.abs(out - ref_img).max())
    print(f"from_pretrained inpaint c{cin}: image max_abs={err:.3e}")
    assert err < 5e-2
    # rejected combinations
    run = dict(height=64, width=64, num_inference_steps=4, guidance_scale=5.0, output_type="np", prompt_embeds=emb)
    with pytest.raises(ValueError, match="starting_image"):
        pipe("x", mask_image=mask[0, 0], **run)
    if cin == 9:
        with pytest.raises(ValueError, match="in_channels=9"):
            pipe("x", **run)
    no_enc = P.from_pretrained(str(tmp_path), height=64, width=64)
    with pytest.raises(ValueError, match="vae_encoder"):
        no_enc("x", starting_image=img, mask_image=mask[0, 0], **run)
    pndm = P.from_pretrained(str(tmp_path), height=64, width=64, with_vae_encoder=True, scheduler_override="PNDM")
    with pytest.raises(ValueError, match="PNDM"):
        pndm("x", starting_image=img, mask_image=mask[0, 0], strength=0.5, **run)


def test_capi_unet_nine_channels_matches_python_engine(cuda_lib):
    from b200sd.capi import CUNet
    from b200sd.model import UNetModel

    sd = config.random_state_dict(config.unet_param_shapes(TINY9), seed=3)
    g = torch.Generator().manual_seed(4)
    x = torch.randn(2, 9, 16, 16, generator=g)
    c = torch.randn(2, TINY9["cross_attention_dim"], 1, 77, generator=g)
    t = torch.tensor([501.0, 21.0])
    h = CUNet(TINY9, sd, batch=2, height=16, width=16)
    out = h.forward(x.half().cuda(), t.cuda(), c.half().cuda()).cpu().numpy()
    py = UNetModel(TINY9, sd, batch=2, height=16, width=16, use_cuda_graph=False)(
        sample=x.half().numpy(), timestep=t.half().numpy(), encoder_hidden_states=c.half().numpy())["noise_pred"]
    diff = float(np.abs(out - py).max())
    print(f"C handle vs Python engine at in_channels = 9: max_abs={diff:.3e} (bitwise: {np.array_equal(out, py)})")
    # as at 4 channels (test_capi_gpu.py): same kernels and order, host-side weight folds summed in another order
    assert diff <= 5e-3
    with torch.no_grad():
        ref = R.unet_forward(sd, TINY9, x, t, c).numpy()
    assert np.abs(out - ref).max() <= 1e-2
    h.close()
