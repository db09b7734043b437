"""GPU tests of the bf16 VAE path (the stock SDXL VAE's activations exceed fp16's range).

Per-launch reference.  Every bf16 GEMM / convolution is compared with an fp64 computation from the bf16 operands the
kernel read: |got - ref| <= r_out * |ref| + tau * B, B = |A| . |W|^T + |bias| + |residual| (the model of
test_gemm_plans_gpu.py).  tau = 2^-14 as there: products of bf16 operands are exact in fp32 and the fp32 accumulation
adds ~2^-24 per addition, random-signed.  r_out is the output rounding.  bf16 has 8 significant bits, so ulp(1) = 2^-7
and round to nearest is within half an ulp: 2^-8 relative, the unit roundoff (fp16: 2^-11).  As the fp16 model takes
r_out = 2^-10 = 2 x 2^-11, this one takes r_out = 2 x 2^-8 = 2^-7; the fp32 value being rounded is itself within
tau * B of ref, so tau * B is charged once more at r_out; 0 for fp32 output.  (2^-9 would be the half-ulp of a 9-bit
significand; bf16 outputs do reach ~2^-8.2 relative error.)  The tolerance must reject the reference with the first or
the last 64-channel k-block left out.

Whole-model bar against the fp32 oracle (TF32 off): PSNR >= 35 dB and max-abs <= 8 x the fp16 full-size bound
(0.02 * max(1, absmax)), i.e. 0.16 * max(1, absmax): 8 = 2^-8 / 2^-11, the ratio of the unit roundoffs."""
import json
import os
import sys

import numpy as np
import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import vae_bf16_fixture as FX  # noqa: E402

pytestmark = pytest.mark.gpu

BF = torch.bfloat16
TAU = 2.0 ** -14
R_OUT = 2.0 ** -7
MODEL_BOUND = 0.16
WIDTHS = (256, 192, 160, 128, 96, 64, 32, 16)


def _taps(x, stride, pad_lo, pad_hi):
    n, h, w, ch = x.shape
    xp = torch.zeros(n, h + pad_lo + pad_hi, w + pad_lo + pad_hi, ch, dtype=x.dtype, device=x.device)
    xp[:, pad_lo:pad_lo + h, pad_lo:pad_lo + w] = x
    ho, wo = h // stride, w // stride
    cols = [xp[:, ty:ty + stride * (ho - 1) + 1:stride, tx:tx + stride * (wo - 1) + 1:stride]
            for ty in range(3) for tx in range(3)]
    return torch.cat(cols, -1).reshape(n * ho * wo, 9 * ch)


def _check_launch(what, a_fn, rows, w, bias, res, out, drop=None):
    """a_fn(r0, r1) -> the fp64 operand rows [r0, r1); chunks of rows keep the fp64 operands small.  Returns the worst
    err / tol; drop = (lo, hi) removes those K columns from the reference (sensitivity check: the worst err / tol
    must then exceed 1)."""
    wd = w.double()
    f32 = out.dtype == torch.float32
    o = out.reshape(rows, -1).double()
    worst = 0.0
    step = max(1, (1 << 27) // max(1, w.shape[1] + w.shape[0]))
    for r0 in range(0, rows, step):
        r1 = min(rows, r0 + step)
        a = a_fn(r0, r1)
        if drop is not None:
            a = a.clone()
            a[:, drop[0]:drop[1]] = 0
        ref = a @ wd.t()
        bound = a.abs() @ wd.abs().t()
        if bias is not None:
            ref += bias.double()
            bound += bias.double().abs()
        if res is not None:
            rr = res.reshape(rows, -1)[r0:r1].double()
            ref += rr
            bound += rr.abs()
        tol = (0.0 if f32 else R_OUT) * ref.abs() + (1.0 if f32 else 1.0 + R_OUT) * TAU * bound + 1e-30
        ratio = (o[r0:r1] - ref).abs() / tol
        worst = max(worst, float(ratio.max()))
    if drop is not None:
        return worst
    assert worst <= 1.0, f"{what}: err/tol {worst:.3f}"
    return worst


def _rand(g, *shape, scale=1.0):
    return (torch.randn(*shape, generator=g, device="cuda") * scale).to(BF)


def _forced_cases():
    cases = []
    for bn in WIDTHS:
        cases.append(("generic", bn))
        if bn >= 32:
            cases += [("plain", bn), ("f32", bn)]
    return cases


@pytest.mark.parametrize("variant,bn", _forced_cases())
def test_forced_bf16_plan_matches_fp64(cuda_lib, variant, bn):
    lib = cuda_lib
    g = torch.Generator(device="cuda").manual_seed(bn * 7 + len(variant))
    if variant == "generic":  # linear, ragged M and N (N % 16 != 0 -> the generic epilogue), residual
        m, c0, n = 300, 200, 2 * bn - 8
        x, w = _rand(g, m, c0), _rand(g, n, c0, scale=c0 ** -0.5)
        bias, res = torch.randn(n, generator=g, device="cuda"), _rand(g, m, n)
        run = lambda: lib.linear(x, w, bias, res, block_n=bn)  # noqa: E731
        a_fn, rows, kdim = (lambda r0, r1: x[r0:r1].double()), m, c0
        desc = dict(mode=0, m=m, n=n, c0=c0, has_residual=True, block_n=bn)
    else:  # convolution: plain = stride 2 + pad_after_only + residual; f32 = stride 1, ragged last tile, fp32 out
        stride = 2 if variant == "plain" else 1
        nimg, h, c0 = 2, 20, 96
        n = 2 * bn if variant == "plain" else bn + 32
        x, w = _rand(g, nimg, h, h, c0), _rand(g, n, 9 * c0, scale=(9 * c0) ** -0.5)
        ho = h // stride
        bias = torch.randn(n, generator=g, device="cuda")
        res = _rand(g, nimg, ho, ho, n) if variant == "plain" else None
        pad = (0, 1) if variant == "plain" else (1, 1)
        f32 = variant == "f32"
        run = lambda: lib.conv3x3(x, w, bias, res, stride=stride, pad_after_only=stride == 2, block_n=bn,  # noqa: E731
                                  out_dtype=torch.float32 if f32 else None)
        taps = _taps(x.double(), stride, *pad)
        a_fn, rows, kdim = (lambda r0, r1: taps[r0:r1]), nimg * ho * ho, 9 * c0
        desc = dict(mode=1, n=n, c0=c0, n_img=nimg, h=h, w=h, stride=stride, has_residual=res is not None,
                    out_f32=f32, pad_after_only=stride == 2, block_n=bn)
    plan = dict(f.split("=") for f in lib.describe_plan(bf16=True, **desc).split())
    assert int(plan["variant"]) == {"generic": 0, "plain": 4, "f32": 3}[variant] and int(plan["block_n"]) == bn, plan
    o1 = run()
    o2 = run()
    torch.cuda.synchronize()
    assert o1.dtype == (torch.float32 if variant == "f32" else BF)
    assert torch.equal(o1.view(torch.int16) if o1.dtype == BF else o1, o2.view(torch.int16) if o2.dtype == BF else o2)
    _check_launch(f"{variant} {bn}", a_fn, rows, w, bias, res, o1)
    last = (kdim - (kdim % 64 or 64), kdim) if variant == "generic" else (kdim - (c0 % 64 or 64), kdim)
    for drop in ((0, 64), last):
        assert _check_launch(f"{variant} {bn} drop", a_fn, rows, w, bias, res, o1, drop=drop) > 1.0, drop


class _Replay:
    """Wraps lib.linear / lib.conv3x3 during a bf16 VAE forward and checks every launch against fp64."""

    def __init__(self, lib):
        self.lib, self.lin0, self.conv0, self.n, self.worst = lib, lib.linear, lib.conv3x3, 0, 0.0

    def linear(self, x, wgt, bias=None, residual=None, **kw):
        assert x.dtype == BF
        xs, ws, rs = x.clone(), wgt.clone(), None if residual is None else residual.clone()
        y = self.lin0(x, wgt, bias, residual, **kw)
        self.n += 1
        self.worst = max(self.worst, _check_launch("linear", lambda r0, r1: xs[r0:r1].double(), xs.shape[0], ws, bias,
                                                   rs, y))
        return y

    def conv3x3(self, x, wgt, bias=None, residual=None, *, stride=1, pad_after_only=False, **kw):
        assert x.dtype == BF
        xs, ws, rs = x.clone(), wgt.clone(), None if residual is None else residual.clone()
        y = self.conv0(x, wgt, bias, residual, stride=stride, pad_after_only=pad_after_only, **kw)
        taps = _taps(xs, stride, 0 if pad_after_only else 1, 1)  # bf16 windows; fp64 per chunk below
        self.n += 1
        self.worst = max(self.worst, _check_launch("conv", lambda r0, r1: taps[r0:r1].double(), taps.shape[0], ws,
                                                   bias, rs, y))
        return y


def _vae_sd(cfg, seed, encoder=False):
    from b200sd import config as C

    shapes = C.vae_encoder_param_shapes(cfg) if encoder else C.vae_decoder_param_shapes(cfg)
    return C.random_state_dict(shapes, seed=seed, dtype=torch.float16)


@pytest.mark.parametrize("which,lat", [("SD_VAE", 64), ("SDXL_VAE", 128), ("encoder", 512)])
def test_every_bf16_vae_launch_matches_fp64(cuda_lib, monkeypatch, which, lat):
    from b200sd import config as C
    from b200sd.vae import VAEDecoderEngine, VAEEncoderEngine

    lib = cuda_lib
    rep = _Replay(lib)
    g = torch.Generator().manual_seed(5)
    if which == "encoder":
        eng = VAEEncoderEngine(C.SDXL_VAE, _vae_sd(C.SDXL_VAE, 8, encoder=True), "cuda", dtype=BF)
        inp = (torch.rand(1, 3, lat, lat, generator=g) * 2 - 1).cuda()
    else:
        cfg = getattr(C, which)
        eng = VAEDecoderEngine(cfg, _vae_sd(cfg, 7), "cuda", dtype=BF)
        inp = torch.randn(1, 4, lat, lat, generator=g).cuda()
    monkeypatch.setattr(lib, "linear", rep.linear)
    monkeypatch.setattr(lib, "conv3x3", rep.conv3x3)
    eng.forward(inp)
    torch.cuda.synchronize()
    print(f"\n{which} {lat}: {rep.n} bf16 launches, worst err/tol {rep.worst:.3f}")
    assert rep.n > 20


@pytest.mark.parametrize("silu", [False, True])
@pytest.mark.parametrize("hw", [32, 256])  # 32^2: cluster kernel; 256^2 x 256 channels: the two-kernel fallback
def test_bf16_group_norm(cuda_lib, hw, silu):
    lib = cuda_lib
    g = torch.Generator(device="cuda").manual_seed(hw)
    c = 256
    x = (torch.randn(2, hw, hw, c, generator=g, device="cuda") * 3e5 + 1e5).to(BF)  # beyond fp16's range
    gamma = 1 + 0.1 * torch.randn(c, generator=g, device="cuda")
    beta = 0.1 * torch.randn(c, generator=g, device="cuda")
    y = lib.group_norm(x, gamma, beta, 32, 1e-6, silu=silu)
    ref = torch.nn.functional.group_norm(x.float().permute(0, 3, 1, 2), 32, gamma, beta, 1e-6)
    if silu:
        ref = torch.nn.functional.silu(ref)
    ref = ref.permute(0, 2, 3, 1)
    assert y.dtype == BF
    err = float((y.float() - ref).abs().max())
    assert err <= 2.0 ** -7 * float(ref.abs().max()) + 1e-3, err


def test_bf16_softmax_latent_prep_nchw_to_nhwc(cuda_lib):
    lib = cuda_lib
    g = torch.Generator(device="cuda").manual_seed(1)
    s = torch.randn(300, 1000, generator=g, device="cuda") * 5
    p = lib.softmax_rows(s, 0.3, out_dtype=BF)
    ref = torch.softmax(s * 0.3, -1)
    assert p.dtype == BF and float(((p.float() - ref).abs() / (ref + 1e-30)).max()) <= 2.0 ** -7
    z = torch.randn(2, 4, 16, 24, generator=g, device="cuda") * 1e5
    w, b = torch.randn(4, 4, generator=g, device="cuda"), torch.randn(4, generator=g, device="cuda")
    o = lib.latent_prep(z, w, b, 0.5, c_pad=8, out_dtype=BF)
    ref = torch.einsum("oc,nchw->nhwo", w, z * 0.5) + b
    assert o.dtype == BF and torch.all(o[..., 4:] == 0)
    assert float((o[..., :4].float() - ref).abs().max()) <= 2.0 ** -7 * float(ref.abs().max()) + 1e-3
    x = torch.randn(2, 3, 17, 9, generator=g, device="cuda") * 1e6
    o = lib.nchw_to_nhwc(x, c_pad=8, out_dtype=BF)
    assert o.dtype == BF and torch.equal(o[..., :3], x.permute(0, 2, 3, 1).to(BF)) and torch.all(o[..., 3:] == 0)
    o2 = lib.nchw_to_nhwc(x, c_pad=8, out=torch.empty_like(o))  # a given output buffer decides the type
    assert o2.dtype == BF and torch.equal(o2, o)
    with pytest.raises(lib.B200SDError):
        lib.linear(o.reshape(-1, 8), torch.zeros(16, 8, dtype=torch.float16, device="cuda"))


def _metrics(got, ref):
    from oracle import restated as R

    err = float((got - ref).abs().max())
    return err, float(R.compute_psnr(got.cpu(), ref.cpu())), float(ref.abs().max())


def _decode_oracle(cfg, sd, z):
    from oracle import restated as R

    with torch.no_grad():
        return R.vae_decode({k: v.cuda().float() for k, v in sd.items()}, cfg, z.cuda()).permute(0, 2, 3, 1)


@pytest.mark.parametrize("which,lat", [("SD_VAE", 64), ("SDXL_VAE", 128)])
def test_bf16_decoder_vs_fp32_oracle(cuda_lib, which, lat):
    from b200sd import config as C
    from b200sd.vae import VAEDecoderEngine

    cfg = getattr(C, which)
    sd = _vae_sd(cfg, 11)
    z = torch.randn(1, 4, lat, lat, generator=torch.Generator().manual_seed(12))
    img = VAEDecoderEngine(cfg, sd, "cuda", dtype=BF).forward(z.cuda())[..., :3]
    ref = _decode_oracle(cfg, sd, z)
    err, psnr, amax = _metrics(img, ref)
    print(f"\nbf16 decoder {which} {8 * lat}^2: max-abs {err:.4f} (bound {MODEL_BOUND * max(1, amax):.4f}), PSNR {psnr:.1f} dB")
    assert psnr >= 35 and err <= MODEL_BOUND * max(1.0, amax)


@pytest.mark.parametrize("size", [512, 1024])
def test_bf16_encoder_vs_fp32_oracle(cuda_lib, size):
    from b200sd import config as C
    from b200sd.vae import VAEEncoderEngine
    from oracle import restated as R

    cfg = C.SDXL_VAE
    sd = _vae_sd(cfg, 13, encoder=True)
    x = torch.rand(1, 3, size, size, generator=torch.Generator().manual_seed(14)) * 2 - 1
    mom = VAEEncoderEngine(cfg, sd, "cuda", dtype=BF).forward(x.cuda())
    with torch.no_grad():
        ref = R.vae_encode({k: v.cuda().float() for k, v in sd.items()}, cfg, x.cuda()).permute(0, 2, 3, 1)
    err, psnr, amax = _metrics(mom, ref)
    print(f"\nbf16 encoder {size}^2: max-abs {err:.4f} (bound {MODEL_BOUND * max(1, amax):.4f}), PSNR {psnr:.1f} dB")
    assert psnr >= 35 and err <= MODEL_BOUND * max(1.0, amax)


def test_overflow_fixture_at_1024(cuda_lib):
    """The scaled weights drive the residual stream past 4 x 65504: the fp16 engine's output is not finite (a plain
    numeric check), the bf16 engine's is and matches the oracle of the unscaled weights."""
    from b200sd import config as C
    from b200sd.vae import VAEDecoderEngine
    from oracle import restated as R

    cfg = C.SDXL_VAE
    sd = _vae_sd(cfg, 15)
    z = torch.randn(1, 4, 128, 128, generator=torch.Generator().manual_seed(16))
    m0, ref = FX.stream_max(R, {k: v.cuda().float() for k, v in sd.items()}, cfg, z.cuda())
    k = FX.pick_k(m0)
    ssd = FX.scaled_state_dict(sd, k)
    ref = ref.permute(0, 2, 3, 1)
    f16 = VAEDecoderEngine(cfg, ssd, "cuda").forward(z.cuda())[..., :3]
    assert not torch.isfinite(f16).all()
    del f16
    img = VAEDecoderEngine(cfg, ssd, "cuda", dtype=BF).forward(z.cuda())[..., :3]
    err, psnr, amax = _metrics(img, ref)
    print(f"\noverflow fixture k={k} (stream {m0:.1f} -> {m0 * 2 ** k:.3g}): bf16 max-abs {err:.4f}, PSNR {psnr:.1f} dB")
    assert torch.isfinite(img).all() and psnr >= 35 and err <= MODEL_BOUND * max(1.0, amax)


def test_bf16_decode_in_cuda_graph_equals_eager(cuda_lib):
    from b200sd import config as C
    from b200sd.vae import VAEDecoderEngine

    eng = VAEDecoderEngine(C.TINY_VAE, _vae_sd(C.TINY_VAE, 17), "cuda", dtype=BF)
    z = torch.randn(1, 4, 32, 32, generator=torch.Generator().manual_seed(18)).cuda()
    eager = eng.forward(z).clone()
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        eng.forward(z)
    torch.cuda.current_stream().wait_stream(s)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        out = eng.forward(z)
    graph.replay()
    torch.cuda.synchronize()
    assert torch.equal(out, eager)


def _write(root, name, sd, cfg):
    st = pytest.importorskip("safetensors.torch")
    os.makedirs(root / name, exist_ok=True)
    st.save_file({k: v.contiguous() for k, v in sd.items()}, str(root / name / "diffusion_pytorch_model.safetensors"))
    (root / name / "config.json").write_text(json.dumps({k: (list(v) if isinstance(v, tuple) else v) for k, v in cfg.items()}))


def _oracle_image(usd, ucfg, vsd, esd, vcfg, emb, pooled, steps, g, lat0=None, img0=None, noise=None,
                  enc_noise=None, strength=0.5):
    """The pipeline's DDIM loop on the oracle (CPU): txt2img from lat0, or image-to-image from img0 (encode with
    enc_noise, noise to timeSteps[start] with `noise`, run the remaining steps), then decode + postprocess."""
    from b200sd import scheduler as S
    from oracle import restated as R

    sched = S.DDIMScheduler(steps)
    abar = R.alphas_cumprod()
    emb = torch.from_numpy(emb).float()
    pooled = torch.from_numpy(pooled).float()
    tid = torch.tensor([[64.0, 64.0, 0.0, 0.0, 64.0, 64.0]] * 2)
    with torch.no_grad():
        start = 0
        if img0 is None:
            x = torch.from_numpy(lat0.astype(np.float32))
        else:
            start = sched.start_step(strength)
            x0 = R.sample_latents(R.vae_encode(esd, vcfg, torch.from_numpy(img0).float()), torch.from_numpy(enc_noise),
                                  vcfg["scaling_factor"])
            x = torch.from_numpy(sched.add_noise(x0.numpy(), noise, strength))
        for t in sched.timesteps[start:]:
            eps = R.unet_forward(usd, ucfg, torch.cat([x, x]).half().float(), torch.tensor([float(t)] * 2), emb,
                                 time_ids=tid, text_embeds=pooled)
            x = R.ddim_step(R.cfg_combine(eps[:1], eps[1:], g), t, x, abar, steps)
        return R.postprocess_image(R.vae_decode(vsd, vcfg, x / vcfg["scaling_factor"])).numpy()


def _image_bar(what, img, ref):
    """The whole-model bar on a postprocessed image: clip(x / 2 + 0.5) halves the decoder's error, so max-abs <=
    MODEL_BOUND / 2 (the decoder output's absmax is ~1 here), and PSNR >= 35 dB."""
    from oracle import restated as R

    err = float(np.abs(img - ref).max())
    psnr = float(R.compute_psnr(torch.from_numpy(img), torch.from_numpy(ref)))
    print(f"\n{what}: image max-abs {err:.4f}, PSNR {psnr:.1f} dB")
    assert psnr >= 35 and err <= MODEL_BOUND / 2, (err, psnr)


@pytest.mark.parametrize("unet,upcast", [("xl", True), ("xl", False), ("xl", None), ("sd2", True)])
def test_from_pretrained_picks_the_vae_dtype(cuda_lib, tmp_path, unet, upcast):
    """force_upcast: true under an SDXL UNet gives bf16 engines: txt2img and img2img through the pipeline match the
    oracle loop.  false / a missing key / an SD-2-shaped UNet keep fp16: decoder and encoder outputs equal directly
    built fp16 models bit for bit."""
    from b200sd import config as C
    from b200sd.pipeline import B200StableDiffusionPipeline
    from b200sd.vae import VAEDecoderModel, VAEEncoderModel

    ucfg = C.TINY_XL_UNET if unet == "xl" else C.TINY_UNET
    usd = C.random_state_dict(C.unet_param_shapes(ucfg), seed=21, dtype=torch.float16)
    _write(tmp_path, "unet", usd, ucfg)
    vcfg = dict(C.TINY_VAE)
    if upcast is not None:
        vcfg["force_upcast"] = upcast
    dsd, esd = _vae_sd(vcfg, 22), _vae_sd(vcfg, 23, encoder=True)
    vsd = dict(dsd, **esd)
    _write(tmp_path, "vae", vsd, vcfg)
    os.makedirs(tmp_path / "scheduler", exist_ok=True)
    (tmp_path / "scheduler" / "scheduler_config.json").write_text(json.dumps({"_class_name": "DDIMScheduler"}))
    pipe = B200StableDiffusionPipeline.from_pretrained(str(tmp_path), height=64, width=64, with_vae_encoder=True)
    want = BF if (unet == "xl" and upcast) else torch.float16
    assert pipe.vae_decoder.engine.dtype == want and pipe.vae_encoder.engine.dtype == want
    zdt = pipe.vae_decoder.expected_inputs["z"]["dtype"]
    assert zdt == (np.float32 if want == BF else np.float16)
    assert pipe.vae_encoder.expected_inputs["x"]["dtype"] == zdt
    z = torch.randn(1, 4, 16, 16, generator=torch.Generator().manual_seed(24))
    got = pipe.vae_decoder(z=z.numpy().astype(zdt))["image"]
    x = (torch.rand(1, 3, 64, 64, generator=torch.Generator().manual_seed(25)) * 2 - 1).numpy()
    if want == BF:
        ref = _decode_oracle(vcfg, dsd, z)
        err, psnr, amax = _metrics(torch.from_numpy(got).permute(0, 2, 3, 1).cuda(), ref)
        assert psnr >= 35 and err <= MODEL_BOUND * max(1.0, amax)
        # end to end: the denoising loop ends in the bf16 decoder (decode_latents), img2img starts in the bf16 encoder
        g = torch.Generator().manual_seed(26)
        emb = torch.randn(2, ucfg["cross_attention_dim"], 1, 77, generator=g).half().numpy()
        pooled = torch.randn(2, ucfg["projection_class_embeddings_input_dim"] - 6 * ucfg["addition_time_embed_dim"],
                             generator=g).numpy()
        steps, gs = 6, 5.0
        lat0 = torch.randn(1, 4, 16, 16, generator=g).half().numpy()
        kw = dict(height=64, width=64, num_inference_steps=steps, guidance_scale=gs, output_type="np",
                  prompt_embeds=emb, pooled_prompt_embeds=pooled)
        img = pipe("x", latents=lat0, **kw).images
        _image_bar("bf16-VAE SDXL txt2img", img, _oracle_image(usd, ucfg, dsd, esd, vcfg, emb, pooled, steps, gs, lat0=lat0))
        np.random.seed(27)
        img = pipe("x", starting_image=x, strength=0.5, **kw).images
        np.random.seed(27)  # the pipeline's draw order: latent noise, then the encoder's noise
        noise = np.random.randn(1, 4, 16, 16).astype(np.float16).astype(np.float32)
        enc_noise = np.random.randn(1, 4, 16, 16).astype(np.float32)
        ref = _oracle_image(usd, ucfg, dsd, esd, vcfg, emb, pooled, steps, gs, img0=x, noise=noise, enc_noise=enc_noise)
        _image_bar("bf16-VAE SDXL img2img", img, ref)
    else:
        direct = VAEDecoderModel(C.TINY_VAE, dsd, batch=1, height=16, width=16)
        assert np.array_equal(got, direct(z=z.numpy().astype(np.float16))["image"])
        denc = VAEEncoderModel(C.TINY_VAE, esd, batch=1, height=64, width=64)
        xh = x.astype(np.float16)
        assert np.array_equal(pipe.vae_encoder(x=xh)["latent"], denc(x=xh)["latent"])
