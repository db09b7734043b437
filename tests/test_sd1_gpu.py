"""GPU tests of Stable Diffusion 1.x: the attention kernel at head dims 40, 80 and 160 against fp32 PyTorch attention,
and the SD-1 UNet, ControlNet and pipeline built on it against the goldens of the unmodified reference
(tests/golden/make_golden_sd1.py) and the oracle.  Tolerances as in test_ops_gpu.py / test_unet_gpu.py."""
import json
import os

import numpy as np
import pytest
import torch

from b200sd import config
from oracle import restated as R

pytestmark = pytest.mark.gpu
GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
MAX_ABS, MIN_PSNR = 1e-2, 35.0
HEAD_DIMS = (40, 80, 160)


def _rand(*shape, seed=0):
    g = torch.Generator(device="cuda").manual_seed(seed)
    return torch.randn(*shape, generator=g, device="cuda").half()


def _close(got, ref, what, atol=3e-3, rtol=3e-3):
    err = (got.float() - ref.float()).abs()
    bad = err > atol + rtol * ref.float().abs()
    assert not bad.any(), f"{what}: {int(bad.sum())}/{bad.numel()} mismatches, max err {err.max().item():.4g}"


def _attn_ref(q, k, v, batch, heads, sq, sk, d, mask=None):
    qh = q.float().reshape(batch, sq, heads, d).permute(0, 2, 1, 3)
    kh = k.float().reshape(batch, sk, heads, d).permute(0, 2, 1, 3)
    vh = v.float().reshape(batch, sk, heads, d).permute(0, 2, 1, 3)
    s = qh @ kh.transpose(-1, -2) * d ** -0.5
    if mask is not None:
        s = s + mask[:, None, None, :]
    return (s.softmax(-1) @ vh).permute(0, 2, 1, 3).reshape(batch * sq, heads * d)


# ------------------------------------------------------------------------------------------------ attention kernel
# SD-1.5 at 512x512: 8 heads; self-attention over 4096 / 1024 / 256 / 64 tokens, cross-attention over 77 text tokens;
# plus a ragged shape whose last query and key tiles are partial
@pytest.mark.parametrize("d", HEAD_DIMS)
@pytest.mark.parametrize("batch,heads,sq,sk", [(2, 8, 4096, 4096), (2, 8, 1024, 1024), (2, 8, 256, 256), (2, 8, 64, 64),
                                               (2, 8, 4096, 77), (2, 8, 256, 77), (2, 8, 64, 77), (1, 3, 200, 333)])
def test_attention_head_dim(cuda_lib, d, batch, heads, sq, sk):
    c = heads * d
    q, k, v = _rand(batch * sq, c, seed=1), _rand(batch * sk, c, seed=2), _rand(batch * sk, c, seed=3)
    out = cuda_lib.attention(q, k, v, batch, heads, sq, sk, d=d)
    _close(out, _attn_ref(q, k, v, batch, heads, sq, sk, d), f"attention d={d} {batch}x{heads}x{sq}x{sk}")


@pytest.mark.parametrize("d", HEAD_DIMS)
def test_attention_head_dim_fused_qkv_and_mask(cuda_lib, d):
    """q, k, v as column views of one [tokens, 3C] GEMM output (the UNet's self-attention) and an additive key mask.
    The output is written into a wider buffer: columns outside [0, heads * d) must stay untouched."""
    batch, heads, s = 2, 8, 200
    c = heads * d
    qkv = _rand(batch * s, 3 * c, seed=1)
    q, k, v = qkv[:, :c], qkv[:, c:2 * c], qkv[:, 2 * c:]
    _close(cuda_lib.attention(q, k, v, batch, heads, s, s, d=d), _attn_ref(q, k, v, batch, heads, s, s, d),
           f"attention d={d} fused-qkv views")
    mask = torch.zeros(batch, s, device="cuda")
    mask[:, 100:] = -1e4
    wide = torch.full((batch * s, c + 64), 7.0, dtype=torch.float16, device="cuda")
    out = cuda_lib.attention(q, k, v, batch, heads, s, s, d=d, mask=mask, out=wide[:, :c])
    _close(out, _attn_ref(q, k, v, batch, heads, s, s, d, mask), f"attention d={d} mask")
    assert bool((wide[:, c:] == 7.0).all()), "attention wrote past the last head's d columns"


@pytest.mark.parametrize("d", HEAD_DIMS)
@pytest.mark.parametrize("batch,heads,sq,sk,masked", [(1, 5, 4096, 4096, False), (2, 5, 4000, 3970, False),
                                                      (1, 5, 4096, 2048, True)])
def test_attention_head_dim_stream_k(cuda_lib, monkeypatch, d, batch, heads, sq, sk, masked):
    """Shapes the stream-K schedule takes (query tiles fill the CTA slots badly): split tiles are merged in slot order, so
    repeated launches are bit-identical, the workspace counters return to zero and the result matches one CTA per tile."""
    c = heads * d
    q, k, v = _rand(batch * sq, c, seed=1), _rand(batch * sk, c, seed=2), _rand(batch * sk, c, seed=3)
    k = (k.float() * torch.linspace(0.5, 6.0, sk, device="cuda").repeat(batch)[:, None]).half()
    mask = None
    if masked:
        mask = torch.zeros(batch, sk, device="cuda")
        mask[:, ::3] = -1e4
    ref = _attn_ref(q, k, v, batch, heads, sq, sk, d, mask)
    out = cuda_lib.attention(q, k, v, batch, heads, sq, sk, d=d, mask=mask)
    _close(out, ref, f"stream-K attention d={d} {batch}x{heads}x{sq}x{sk}")
    for _ in range(2):
        assert torch.equal(out, cuda_lib.attention(q, k, v, batch, heads, sq, sk, d=d, mask=mask))
    ws = cuda_lib._attention_workspace(q.device, d)
    assert ws.numel() >= cuda_lib.load().b200sd_attention_workspace_bytes_for(d)
    assert int(ws[:65536].max()) == 0
    monkeypatch.setenv("B200SD_ATTN_STREAMK", "0")
    whole = cuda_lib.attention(q, k, v, batch, heads, sq, sk, d=d, mask=mask)
    monkeypatch.delenv("B200SD_ATTN_STREAMK")
    _close(whole, ref, f"one CTA per query tile d={d}")
    assert (out.float() - whole.float()).abs().max().item() <= 2e-3


def test_attention_rejects_other_head_dims(cuda_lib):
    q = _rand(128, 2 * 48)
    with pytest.raises(cuda_lib.B200SDError, match="head dim 48"):
        cuda_lib.attention(q, q, q, 1, 2, 128, 128, d=48)
    assert cuda_lib.load().b200sd_attention_workspace_bytes_for(48) == 0
    assert cuda_lib.load().b200sd_attention_workspace_bytes_for(64) == cuda_lib.load().b200sd_attention_workspace_bytes()


# ------------------------------------------------------------------------------------------------ UNet / ControlNet
def _inputs(cfg, seed, batch=2, seq=77):
    g = torch.Generator().manual_seed(seed)
    s = cfg["sample_size"]
    return (torch.randn(batch, cfg["in_channels"], s, s, generator=g),
            torch.randn(batch, cfg["cross_attention_dim"], 1, seq, generator=g))


def _fingerprint(sd):
    keys = sorted(sd.keys())
    picks = [keys[0], keys[len(keys) // 2], keys[-1]]
    return np.array([float(sd[k].double().sum()) for k in picks] + [float(len(keys))])


def _check(out, ref, what, max_abs=MAX_ABS):
    err = float(np.abs(out - ref).max())
    psnr = R.compute_psnr(torch.from_numpy(np.asarray(out, np.float32)), torch.from_numpy(np.asarray(ref, np.float32)))
    print(f"{what}: max_abs={err:.3e} psnr={psnr:.1f} dB (ref absmax {np.abs(ref).max():.3f})")
    assert np.isfinite(out).all(), what
    assert err <= max_abs and psnr >= MIN_PSNR, f"{what}: max_abs={err:.3e} psnr={psnr:.1f}"


@pytest.mark.parametrize("impl", ["ORIGINAL", "SPLIT_EINSUM", "SPLIT_EINSUM_V2"])
def test_unet_tiny_sd1_vs_reference_golden(cuda_lib, impl):
    """Down blocks at head dims 40 / 80, mid block 160, up blocks 80 / 40."""
    from b200sd import unet as U
    from b200sd.model import UNetModel

    U.ATTENTION_IMPLEMENTATION_IN_EFFECT = U.AttentionImplementations[impl]
    try:
        cfg = config.TINY_SD1_UNET
        gold = np.load(os.path.join(GOLD, "unet_tiny_sd1.npz"))
        sd = config.random_state_dict(config.unet_param_shapes(cfg), seed=int(gold["weight_seed"]))
        x, c = _inputs(cfg, int(gold["input_seed"]))
        t = np.array([float(gold["timestep"])] * 2, np.float16)
        kw = dict(sample=x.half().numpy(), timestep=t, encoder_hidden_states=c.half().numpy())
        eager = UNetModel(cfg, sd, batch=2, height=16, width=16, use_cuda_graph=False)(**kw)["noise_pred"]
        _check(eager, gold[f"noise_pred_{impl}"], f"tiny SD-1 unet vs reference golden [{impl}]")
        graph = UNetModel(cfg, sd, batch=2, height=16, width=16, use_cuda_graph=True)
        g1 = graph(**kw)["noise_pred"]
        assert np.array_equal(eager, g1) and np.array_equal(g1, graph(**kw)["noise_pred"])
    finally:
        U.ATTENTION_IMPLEMENTATION_IN_EFFECT = U.AttentionImplementations["SPLIT_EINSUM"]


def test_unet_sd15_vs_reference_golden(cuda_lib):
    """Full-size SD-1.5 UNet, batch 2, 64x64 latents, through the Python engine and the C ABI."""
    from b200sd.capi import CUNet
    from b200sd.model import UNetModel

    cfg = config.SD15_UNET
    gold = np.load(os.path.join(GOLD, "unet_sd15.npz"))
    sd = config.random_state_dict(config.unet_param_shapes(cfg), seed=int(gold["weight_seed"]))
    assert np.allclose(_fingerprint(sd), gold["fingerprint"], rtol=1e-6), "weight generator drifted"
    x, c = _inputs(cfg, int(gold["input_seed"]))
    t = float(gold["timestep"])
    m = UNetModel(cfg, sd, batch=2, height=64, width=64, use_cuda_graph=True)
    out = m(sample=x.half().numpy(), timestep=np.array([t, t], np.float16),
            encoder_hidden_states=c.half().numpy())["noise_pred"]
    _check(out, gold["noise_pred_ORIGINAL"], "SD-1.5 unet vs reference golden")
    del m
    h = CUNet(cfg, sd, batch=2, height=64, width=64)
    try:
        cout = h.forward(x.half().cuda(), torch.tensor([t, t]).cuda(), c.half().cuda()).cpu().numpy()
    finally:
        h.close()
    _check(cout, gold["noise_pred_ORIGINAL"], "C-ABI SD-1.5 unet vs reference golden")


def test_controlnet_tiny_sd1_vs_reference_golden_and_chain_into_unet(cuda_lib):
    from b200sd.controlnet import ControlNetModel
    from b200sd.model import UNetModel

    gold = np.load(os.path.join(GOLD, "controlnet_tiny_sd1.npz"))
    ccfg = config.TINY_SD1_CONTROLNET
    csd = config.random_state_dict(config.controlnet_param_shapes(ccfg), seed=int(gold["weight_seed"]))
    x, c = _inputs(config.TINY_SD1_UNET, int(gold["input_seed"]))
    cond = torch.rand(2, 3, 128, 128, generator=torch.Generator().manual_seed(int(gold["cond_seed"])))
    t = np.array([501.0, 501.0], np.float16)
    cn = ControlNetModel(ccfg, csd, batch=2, height=16, width=16)
    res = cn(sample=x.half().numpy(), timestep=t, encoder_hidden_states=c.half().numpy(),
             controlnet_cond=cond.half().numpy())
    st = int(gold["stride"])
    n = len([k for k in gold.files if k.startswith("residual_")])
    assert len(res) == n == 7
    for i in range(n):
        ref = gold[f"residual_{i}"].astype(np.float32)
        got = res[f"additional_residual_{i}"][:, :, ::st, ::st]
        _check(got, ref, f"SD-1 controlnet residual {i}", max_abs=1e-2 * max(1.0, float(np.abs(ref).max())))
    ucfg = dict(config.TINY_SD1_UNET, support_controlnet=True)
    usd = config.random_state_dict(config.unet_param_shapes(ucfg), seed=5)
    unet = UNetModel(ucfg, usd, batch=2, height=16, width=16, use_cuda_graph=False)
    kw = {k: v.astype(np.float16) for k, v in res.items()}
    out = unet(sample=x.half().numpy(), timestep=t, encoder_hidden_states=c.half().numpy(), **kw)["noise_pred"]
    rres = [torch.from_numpy(res[f"additional_residual_{i}"].astype(np.float16).astype(np.float32)) for i in range(n)]
    with torch.no_grad():
        uref = R.unet_forward(usd, ucfg, x, torch.tensor([501.0, 501.0]), c, additional_residuals=rres).numpy()
    _check(out, uref, "SD-1 controlnet -> control-unet chain")


# ------------------------------------------------------------------------------------------------ pipeline
def _write_sd1_dir(root, ucfg, tcfg, seed):
    st = pytest.importorskip("safetensors.torch")
    comps = {"unet": (config.random_state_dict(config.unet_param_shapes(ucfg), seed=seed, dtype=torch.float16), ucfg,
                      "UNet2DConditionModel", "diffusion_pytorch_model.safetensors"),
             "vae": (config.random_state_dict(config.vae_decoder_param_shapes(config.TINY_VAE), seed=seed + 1,
                                              dtype=torch.float16), config.TINY_VAE, "AutoencoderKL",
                     "diffusion_pytorch_model.safetensors"),
             "text_encoder": (config.random_clip_text_state_dict(tcfg, seed=seed + 2, dtype=torch.float16), tcfg,
                              "CLIPTextModel", "model.safetensors")}
    for name, (sd, cfg, cls, fname) in comps.items():
        os.makedirs(root / name, exist_ok=True)
        st.save_file({k: v.contiguous() for k, v in sd.items()}, str(root / name / fname))
        meta = {k: (list(v) if isinstance(v, tuple) else v) for k, v in cfg.items()}
        (root / name / "config.json").write_text(json.dumps(dict(meta, _class_name=cls)))
    vocab = {"<|startoftext|>": 998, "<|endoftext|>": 999, "red</w>": 2, "cu": 3, "be</w>": 4, "c": 5, "u": 6}
    os.makedirs(root / "tokenizer", exist_ok=True)
    (root / "tokenizer" / "merges.txt").write_text("#version: 0.2\nc u\nb e</w>\nr e\nre d</w>\n")
    (root / "tokenizer" / "vocab.json").write_text(json.dumps(vocab))
    os.makedirs(root / "scheduler", exist_ok=True)
    (root / "scheduler" / "scheduler_config.json").write_text(json.dumps({"_class_name": "PNDMScheduler"}))
    return {k: v[0] for k, v in comps.items()}


def test_from_pretrained_sd1_directory_equals_direct_construction(cuda_lib, tmp_path):
    """An SD-1-shaped diffusers directory: integer attention_head_dim (8 heads: d = 40 / 80), 1x1-conv proj_in, a
    CLIP-L-shaped text encoder (quick-GELU, no projection, last_hidden_state) and the PNDM scheduler."""
    from b200sd.model import UNetModel
    from b200sd.pipeline import B200StableDiffusionPipeline
    from b200sd.text_encoder import TextEncoderModel
    from b200sd.vae import VAEDecoderModel

    tcfg = dict(config.TINY_CLIP_TEXT, hidden_act="quick_gelu")
    ucfg = dict(config.TINY_SD1_UNET, attention_head_dim=8, cross_attention_dim=tcfg["hidden_size"])
    sds = _write_sd1_dir(tmp_path, ucfg, tcfg, seed=61)
    assert sds["unet"]["down_blocks.0.attentions.0.proj_in.weight"].dim() == 4
    pipe = B200StableDiffusionPipeline.from_pretrained(str(tmp_path), height=64, width=64)
    assert pipe.scheduler_name == "PNDM" and not pipe.xl and pipe.text_encoder is not None
    direct = B200StableDiffusionPipeline(UNetModel(ucfg, sds["unet"], batch=2, height=16, width=16),
                                         VAEDecoderModel(config.TINY_VAE, sds["vae"], batch=1, height=16, width=16),
                                         scheduler="PNDM", text_encoder=TextEncoderModel(tcfg, sds["text_encoder"], batch=1),
                                         tokenizer=pipe.tokenizer, force_zeros_for_empty_prompt=False)
    kw = dict(height=64, width=64, num_inference_steps=4, guidance_scale=5.0, output_type="np", seed=7, rng="torch")
    a = pipe("red cube", **kw).images
    b = direct("red cube", **kw).images
    assert a.shape == (1, 64, 64, 3) and np.isfinite(a).all() and np.array_equal(a, b)


def test_pipeline_tiny_sd1_end_to_end_vs_oracle(cuda_lib):
    """DDIM txt2img from a text prompt with the SD-1-shaped UNet vs the same loop run with the oracle on the CPU."""
    from b200sd import scheduler as S
    from b200sd.pipeline import B200StableDiffusionPipeline

    ucfg, vcfg = config.TINY_SD1_UNET, config.TINY_VAE
    pipe = B200StableDiffusionPipeline.from_random_init("tiny", unet_cfg=ucfg, images_per_call=1, height=64, width=64,
                                                        seed=13)
    np.random.seed(95)
    lat0 = np.random.randn(1, 4, 16, 16).astype(np.float16)
    steps, g, prompt = 5, 7.5, "a photo of an astronaut riding a horse"
    img = pipe(prompt, height=64, width=64, num_inference_steps=steps, guidance_scale=g, latents=lat0,
               output_type="np").images
    assert img.shape == (1, 64, 64, 3)
    usd = config.random_state_dict(config.unet_param_shapes(ucfg), seed=13, dtype=torch.float16)
    vsd = config.random_state_dict(config.vae_decoder_param_shapes(vcfg), seed=14, dtype=torch.float16)
    emb = torch.from_numpy(pipe._encode_prompt([prompt], True, None)).float()
    x = torch.from_numpy(lat0.astype(np.float32))
    abar = R.alphas_cumprod()
    with torch.no_grad():
        for t in S.DDIMScheduler(steps).timesteps:
            eps = R.unet_forward(usd, ucfg, torch.cat([x, x]).half().float(), torch.tensor([float(t)] * 2), emb)
            x = R.ddim_step(R.cfg_combine(eps[:1], eps[1:], g), t, x, abar, steps)
        ref = R.postprocess_image(R.vae_decode(vsd, vcfg, x / 0.18215)).numpy()
    err = float(np.abs(img - ref).max())
    print(f"pipeline tiny SD-1: image max_abs={err:.3e}")
    assert err < 3e-2
