"""GPU tests of ControlNet with SDXL: the scaled residual-injection kernel against torch's fp16 arithmetic, the SDXL
ControlNet engine against the goldens of the reference modules (make_golden_controlnet_xl.py) and the restatement of controlnet_xl_oracle.py,
the device loop with conditioning scales and guidance windows against the oracle loop, and every launch of the SDXL
ControlNet against its fp64 reference (the replays of test_gemm_plans_gpu.py / test_op_launches_gpu.py)."""
import json
import os
import sys

import numpy as np
import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import controlnet_xl_oracle as CX  # noqa: E402
import model_cases as MC  # noqa: E402
import test_gemm_plans_gpu as TG  # noqa: E402
import test_op_launches_gpu as TO  # noqa: E402
import test_unet_gpu as TU  # noqa: E402

from b200sd import config  # noqa: E402
from b200sd import scheduler as S  # noqa: E402
from oracle import restated as R  # noqa: E402

pytestmark = pytest.mark.gpu

GOLD = os.path.join(os.path.dirname(__file__), "golden")


# ------------------------------------------------------------------------------------------------ injection kernel
def _emulate(skip, res, scales):
    """diffusers' fp16 order with torch fp16 ops: t = s_0 r_0, t = t + s_k r_k, skip + t."""
    t = res[0] * scales[0]
    for r, s in zip(res[1:], scales[1:]):
        t = t + r * s
    return t if skip is None else skip + t


@pytest.mark.parametrize("numel", [8 * 4099, 8 * 4099 + 5])
@pytest.mark.parametrize("scales", [(1.0,), (0.5,), (0.0,), (-0.7, 2.5), (1.0, 1.0), (0.5, 0.0, 2.5), (1.0, 1.0, 1.0),
                                    (2.5, -0.7, 0.5)])
def test_control_inject_matches_torch_fp16(cuda_lib, numel, scales):
    L = cuda_lib
    g = torch.Generator(device="cuda").manual_seed(numel + len(scales))
    mk = lambda: (torch.randn(numel, generator=g, device="cuda") * 3).half()  # noqa: E731
    skip, res = mk(), [mk() for _ in scales]
    sc = torch.tensor(scales, dtype=torch.float32, device="cuda")
    out = L.control_inject(skip, res, sc)
    assert torch.equal(out, _emulate(skip, res, scales)), float((out.float() - _emulate(skip, res, scales).float()).abs().max())
    assert torch.equal(L.control_inject(None, res, sc), _emulate(None, res, scales))
    if all(s == 1.0 for s in scales):  # the launches the SD ControlNet paths made before: bit for bit
        e = numel - numel % 2  # b200sd_add takes an even number of elements
        sk, rs = skip[:e], [r[:e] for r in res]
        if len(rs) == 1:
            want = L.add(sk, rs[0])
        elif len(rs) == 2:
            want = L.add(sk, L.add(rs[0], rs[1]))
        else:
            want = L.add(sk, L.add(L.add(rs[0], rs[1]), rs[2]))
        assert torch.equal(out[:e], want)
    # a misaligned view takes the element-wise path and gives the same bits
    off = L.control_inject(skip[1:], [r[1:] for r in res], sc)
    assert torch.equal(off, _emulate(skip[1:], [r[1:] for r in res], scales))
    # the scales are read on the device: a captured launch replays with new values
    buf = torch.empty_like(skip)
    gr = torch.cuda.CUDAGraph()
    torch.cuda.synchronize()
    with torch.cuda.graph(gr):
        L.control_inject(skip, res, sc, out=buf)
    new = [s * 0.25 - 1.0 for s in scales]
    sc.copy_(torch.tensor(new))
    gr.replay()
    torch.cuda.synchronize()
    assert torch.equal(buf, _emulate(skip, res, new))


# ------------------------------------------------------------------------------------------------ engine parity
def _gold_inputs(gold, cfg):
    size = int(gold["size"])
    pooled = cfg["projection_class_embeddings_input_dim"] - 6 * cfg["addition_time_embed_dim"]
    g = torch.Generator().manual_seed(int(gold["input_seed"]))
    x = torch.randn(2, 4, size, size, generator=g)
    ctx = torch.randn(2, cfg["cross_attention_dim"], 1, 77, generator=g)
    te = torch.randn(2, pooled, generator=g)
    cond = torch.rand(2, 3, 8 * size, 8 * size, generator=torch.Generator().manual_seed(int(gold["cond_seed"])))
    return x, ctx, te, torch.from_numpy(gold["time_ids"]), cond


@pytest.mark.parametrize("name,cfg_name,fp16", [("controlnet_tiny_xl", "TINY_XL_CONTROLNET", False),
                                                 ("controlnet_sdxl", "SDXL_CONTROLNET", True)])
def test_sdxl_controlnet_vs_reference_golden(cuda_lib, name, cfg_name, fp16):
    from b200sd.controlnet import ControlNetModel
    gold = np.load(os.path.join(GOLD, f"{name}.npz"))
    cfg = getattr(config, cfg_name)
    sd = config.random_state_dict(config.controlnet_param_shapes(cfg), seed=int(gold["weight_seed"]),
                                  dtype=torch.float16 if fp16 else torch.float32)
    x, ctx, te, tid, cond = _gold_inputs(gold, cfg)
    size, st = int(gold["size"]), int(gold["stride"])
    m = ControlNetModel(cfg, sd, batch=2, height=size, width=size)
    assert set(m.expected_inputs) >= {"time_ids", "text_embeds"}
    out = m(sample=x.half().numpy(), timestep=np.array([501.0, 501.0], np.float16),
            encoder_hidden_states=ctx.half().numpy(), controlnet_cond=cond.half().numpy(),
            time_ids=tid.half().numpy(), text_embeds=te.half().numpy())
    n = len([k for k in gold.files if k.startswith("residual_")])
    assert len(out) == n == (10 if cfg_name == "SDXL_CONTROLNET" else 7)
    for i in range(n):
        ref = gold[f"residual_{i}"].astype(np.float32)
        TU._check(out[f"additional_residual_{i}"][:, :, ::st, ::st], ref, f"{name} residual {i} (reference golden)",
                  max_abs=1e-2 * max(1.0, float(np.abs(ref).max())))


def _sdxl_inputs(h, w, seed):
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(2, 4, h, w, generator=g).half()
    ctx = torch.randn(2, 2048, 1, 77, generator=g).half()
    te = torch.randn(2, 1280, generator=g).half()
    tid = torch.tensor([[8.0 * h, 8.0 * w, 0.0, 0.0, 8.0 * h, 8.0 * w]] * 2).half()
    cond = torch.rand(2, 3, 8 * h, 8 * w, generator=g).half()
    return x, ctx, te, tid, cond


def test_sdxl_controlnet_1024_vs_oracle_and_chain_into_unet(cuda_lib):
    """SDXL ControlNet at 1024x1024 (128x128 latents) against the restatement (controlnet_xl_oracle.py) run on the device in fp32, at the bar
    of test_controlnet_sd21_vs_reference_golden; then its residuals chained into the SDXL UNet (32x32 latents) against
    restated.unet_forward with the same residuals."""
    from b200sd.controlnet import ControlNetModel
    from b200sd.model import UNetModel
    cfg = config.SDXL_CONTROLNET
    sd = config.random_state_dict(config.controlnet_param_shapes(cfg), seed=81, dtype=torch.float16)
    x, ctx, te, tid, cond = _sdxl_inputs(128, 128, 82)
    t = np.array([501.0, 501.0], np.float16)
    m = ControlNetModel(cfg, sd, batch=2, height=128, width=128, use_cuda_graph=False)
    out = m(sample=x.numpy(), timestep=t, encoder_hidden_states=ctx.numpy(), controlnet_cond=cond.numpy(),
            time_ids=tid.numpy(), text_embeds=te.numpy())
    del m
    dev = {k: v.cuda().float() for k, v in sd.items()}
    with torch.no_grad():
        live = CX.controlnet_forward_xl(dev, cfg, x.cuda().float(), torch.tensor([501.0, 501.0], device="cuda"),
                                        ctx.cuda().float(), cond.cuda().float(), tid.cuda().float(), te.cuda().float())
    assert len(live) == len(out) == 10
    for i, r in enumerate(live):
        TU._check(out[f"additional_residual_{i}"], r.cpu().numpy(), f"SDXL controlnet 1024 residual {i}")
    del dev, live, out
    torch.cuda.empty_cache()
    # chained into the SDXL UNet
    x, ctx, te, tid, cond = _sdxl_inputs(32, 32, 83)
    cn = ControlNetModel(cfg, sd, batch=2, height=32, width=32)
    res = cn(sample=x.numpy(), timestep=t, encoder_hidden_states=ctx.numpy(), controlnet_cond=cond.numpy(),
             time_ids=tid.numpy(), text_embeds=te.numpy())
    ucfg = dict(config.SDXL_BASE_UNET, support_controlnet=True)
    usd = config.random_state_dict(config.unet_param_shapes(ucfg), seed=84, dtype=torch.float16)
    u = UNetModel(ucfg, usd, batch=2, height=32, width=32)
    kw = {k: v.astype(np.float16) for k, v in res.items()}
    y = u(sample=x.numpy(), timestep=t, encoder_hidden_states=ctx.numpy(), time_ids=tid.numpy(),
          text_embeds=te.numpy(), **kw)["noise_pred"]
    del u
    dev = {k: v.cuda().float() for k, v in usd.items()}
    rr = [torch.from_numpy(res[f"additional_residual_{i}"]).cuda().half().float() for i in range(10)]
    with torch.no_grad():
        ref = R.unet_forward(dev, ucfg, x.cuda().float(), torch.tensor([501.0, 501.0], device="cuda"),
                             ctx.cuda().float(), tid.cuda().float(), te.cuda().float(), additional_residuals=rr)
    TU._check(y, ref.cpu().numpy(), "SDXL controlnet -> SDXL UNet chain")


# ------------------------------------------------------------------------------------------------ pipeline
STEPS, G = 4, 5.0


def _tiny_xl_pipe(n_nets, seed=21):
    from b200sd.pipeline import B200StableDiffusionPipeline
    return B200StableDiffusionPipeline.from_random_init("tiny", unet_cfg=config.TINY_XL_UNET, height=64, width=64,
                                                        seed=seed, controlnet_cfgs=[config.TINY_XL_CONTROLNET] * n_nets)


def _loop_inputs(pipe, n_nets):
    rs = np.random.RandomState(5)
    emb = (rs.standard_normal((2, 96, 1, 77)) * 0.5).astype(np.float16)
    lat = rs.standard_normal((1, 4, 16, 16)).astype(np.float32)
    tid = torch.tensor([[64.0, 64.0, 0.0, 0.0, 64.0, 64.0]] * 2, device="cuda")
    te = torch.from_numpy(rs.standard_normal((2, 64)).astype(np.float32)).cuda()
    conds = [rs.rand(3, 128, 128).astype(np.float16) for _ in range(n_nets)]
    return emb, lat, tid, te, pipe.prepare_control_cond(conds, True, 1, 1)


def _oracle_loop(n_nets, emb, lat, tid, te, cc, scales, starts, ends, guided=True, seed=21):
    from b200sd.pipeline import controlnet_keep
    ucfg = dict(config.TINY_XL_UNET, support_controlnet=True)
    ccfg = config.TINY_XL_CONTROLNET
    usd = config.random_state_dict(config.unet_param_shapes(ucfg), seed=seed, dtype=torch.float16)
    csds = [config.random_state_dict(config.controlnet_param_shapes(ccfg), seed=seed + 2 + k, dtype=torch.float16)
            for k in range(n_nets)]
    sl = slice(0, 2) if guided else slice(1, 2)
    emb = torch.from_numpy(emb).float()[sl]
    tid, te = tid.cpu()[sl], te.cpu()[sl]
    conds = [torch.from_numpy(c).float()[sl] for c in cc]
    x = torch.from_numpy(lat)
    abar = R.alphas_cumprod()
    keep = controlnet_keep(STEPS, starts, ends)
    with torch.no_grad():
        for i, t in enumerate(S.DDIMScheduler(STEPS).timesteps):
            xin = (torch.cat([x, x]) if guided else x).half().float()
            tt = torch.tensor([float(t)] * xin.shape[0])
            res = None
            for k in keep[i]:
                r = CX.controlnet_forward_xl(csds[k], ccfg, xin, tt, emb, conds[k], tid, te)
                res = [scales[k] * a for a in r] if res is None else [b + scales[k] * a for a, b in zip(r, res)]
            eps = R.unet_forward(usd, ucfg, xin, tt, emb, tid, te, additional_residuals=res)
            if guided:
                eps = R.cfg_combine(eps[:1], eps[1:], G)
            x = R.ddim_step(eps, t, x, abar, STEPS)
    return x.numpy()


@pytest.mark.parametrize("n_nets", [1, 2])
def test_tiny_xl_loop_with_scales_and_window_vs_oracle(cuda_lib, n_nets):
    """Scales (0.7, 0.3) and, on the last net, the window [0, 0.5]: the eager loop against the oracle loop; the loop
    graph bit-identical to the eager loop; scale 0 on every net bit-identical to no conditions; new scales replay the
    same captured graph and match the eager loop at those scales."""
    pipe = _tiny_xl_pipe(n_nets)
    emb, lat, tid, te, cc = _loop_inputs(pipe, n_nets)
    scales, starts, ends = [0.7, 0.3][:n_nets], [0.0] * n_nets, [1.0] * (n_nets - 1) + [0.5]
    kw = dict(time_ids=tid, text_embeds=te, controlnet_cond=cc, controlnet_conditioning_scale=scales,
              control_guidance_start=starts, control_guidance_end=ends)
    rec = []
    eager = pipe.denoise(emb, lat, STEPS, G, record=rec, **kw).clone()
    ref = _oracle_loop(n_nets, emb, lat, tid, te, cc, scales, starts, ends)
    TU._check(eager.cpu().numpy(), ref, f"tiny-XL loop, {n_nets} ControlNet(s)", max_abs=2e-2 * max(1.0, float(np.abs(ref).max())))
    graph = pipe.denoise(emb, lat, STEPS, G, **kw).clone()
    assert torch.equal(graph, eager), float((graph - eager).abs().max())
    assert len(pipe._loop_graphs) == 1
    # new scales: the same graph, the eager loop's bits at those scales
    kw2 = dict(kw, controlnet_conditioning_scale=[-0.4, 1.3][:n_nets])
    graph2 = pipe.denoise(emb, lat, STEPS, G, **kw2).clone()
    assert len(pipe._loop_graphs) == 1
    eager2 = pipe.denoise(emb, lat, STEPS, G, record=[], **kw2).clone()
    assert torch.equal(graph2, eager2) and not torch.equal(graph2, graph)
    # scale 0 everywhere == called without conditions
    zero = pipe.denoise(emb, lat, STEPS, G, **dict(kw, controlnet_conditioning_scale=0.0)).clone()
    plain = pipe.denoise(emb, lat, STEPS, G, time_ids=tid, text_embeds=te).clone()
    assert torch.equal(zero, plain), float((zero - plain).abs().max())


def test_tiny_xl_guidance_free_loop_with_controlnet_vs_oracle(cuda_lib):
    pipe = _tiny_xl_pipe(1)
    emb, lat, tid, te, cc = _loop_inputs(pipe, 1)
    kw = dict(time_ids=tid, text_embeds=te, controlnet_cond=cc, controlnet_conditioning_scale=0.5)
    graph = pipe.denoise(emb, lat, STEPS, 1.0, **kw).clone()
    ref = _oracle_loop(1, emb, lat, tid, te, cc, [0.5], [0.0], [1.0], guided=False)
    TU._check(graph.cpu().numpy(), ref, "tiny-XL guidance-free loop + ControlNet",
              max_abs=2e-2 * max(1.0, float(np.abs(ref).max())))
    eager = pipe.denoise(emb, lat, STEPS, 1.0, record=[], **kw).clone()
    assert torch.equal(graph, eager)


def _write_component(root, sd, cfg, cls):
    st = pytest.importorskip("safetensors.torch")
    os.makedirs(root, exist_ok=True)
    st.save_file({k: v.contiguous() for k, v in sd.items()}, str(root / "diffusion_pytorch_model.safetensors"))
    meta = {k: (list(v) if isinstance(v, tuple) else v) for k, v in cfg.items()}
    meta["_class_name"] = cls
    (root / "config.json").write_text(json.dumps(meta))


def test_from_pretrained_sdxl_with_controlnet_equals_direct_construction(cuda_lib, tmp_path):
    from b200sd.controlnet import ControlNetModel
    from b200sd.model import UNetModel
    from b200sd.pipeline import B200StableDiffusionPipeline as P
    from b200sd.vae import VAEDecoderModel
    ucfg, vcfg, ccfg = config.TINY_XL_UNET, config.TINY_VAE, config.TINY_XL_CONTROLNET
    usd = config.random_state_dict(config.unet_param_shapes(ucfg), seed=31, dtype=torch.float16)
    vsd = config.random_state_dict(config.vae_decoder_param_shapes(vcfg), seed=32, dtype=torch.float16)
    csd = config.random_state_dict(config.controlnet_param_shapes(ccfg), seed=33, dtype=torch.float16)
    _write_component(tmp_path / "sdxl" / "unet", usd, ucfg, "UNet2DConditionModel")
    _write_component(tmp_path / "sdxl" / "vae", vsd, vcfg, "AutoencoderKL")
    os.makedirs(tmp_path / "sdxl" / "scheduler")
    (tmp_path / "sdxl" / "scheduler" / "scheduler_config.json").write_text(json.dumps({"_class_name": "DDIMScheduler"}))
    _write_component(tmp_path / "cn", csd, dict(ccfg, global_pool_conditions=False), "ControlNetModel")
    loaded = P.from_pretrained(str(tmp_path / "sdxl"), controlnet_dirs=[str(tmp_path / "cn")], height=64, width=64)
    direct = P(UNetModel(dict(ucfg, support_controlnet=True), usd, batch=2, height=16, width=16),
               VAEDecoderModel(vcfg, vsd, batch=1, height=16, width=16), scheduler="DDIM", xl=True,
               controlnet=[ControlNetModel(ccfg, csd, batch=2, height=16, width=16)])
    emb, lat, tid, te, cc = _loop_inputs(direct, 1)
    kw = dict(time_ids=tid, text_embeds=te, controlnet_cond=cc, controlnet_conditioning_scale=0.5)
    a = loaded.denoise(emb, lat, STEPS, G, **kw).clone()
    b = direct.denoise(emb, lat, STEPS, G, **kw).clone()
    assert torch.isfinite(a).all() and torch.equal(a, b)
    # a ControlNet of another base model is refused before any weights are read
    bad = tmp_path / "cn_sd"
    os.makedirs(bad)
    (bad / "config.json").write_text(json.dumps({k: (list(v) if isinstance(v, tuple) else v)
                                                 for k, v in config.TINY_CONTROLNET.items()}))
    with pytest.raises(ValueError, match="cross_attention_dim|block_out_channels|down_block_types"):
        P.from_pretrained(str(tmp_path / "sdxl"), controlnet_dirs=[str(bad)], height=64, width=64)


# ------------------------------------------------------------------------------------------------ per-launch replays
@pytest.mark.parametrize("hw", [(128, 128), (96, 168)], ids=["1024x1024", "768x1344"])
def test_sdxl_controlnet_launches_match_fp64_reference(cuda_lib, monkeypatch, hw):
    """Every GEMM / convolution launch, then every other launch, of the SDXL ControlNet at 1024x1024 and at the
    768x1344 aspect-ratio bucket against the fp64 reference of that one launch."""
    from b200sd.controlnet import ControlNetModel
    lib = cuda_lib
    for k in ("B200SD_CLUSTER_SPLITK", "B200SD_STAGED", "B200SD_FUSED", "B200SD_HALO_TMA"):
        monkeypatch.delenv(k, raising=False)
    cfg = config.SDXL_CONTROLNET
    sd = config.random_state_dict(config.controlnet_param_shapes(cfg), seed=6, dtype=torch.float16)
    m = ControlNetModel(cfg, sd, batch=2, height=hw[0], width=hw[1], use_cuda_graph=False)
    name = f"controlnet_sdxl_{8 * hw[0]}x{8 * hw[1]}"
    inputs = MC.model_inputs(m, seed=9)
    with monkeypatch.context() as mp:
        rep = TG._Replay(lib, name)
        mp.setattr(lib, "linear", rep.linear)
        mp.setattr(lib, "conv3x3", rep.conv3x3)
        m(**inputs)
        torch.cuda.synchronize()
        print(f"\n{rep.report()}")
        assert rep.plans, "no GEMM / convolution launch was seen"
    with monkeypatch.context() as mp:
        rep = TO._Replay(lib, name)
        rep.install(mp)
        m(**inputs)
        torch.cuda.synchronize()
        print(f"\n{rep.report()}")
        ops = {key[0] for key in rep.rows}
        assert {"attention", "group_norm", "linear_small", "timestep_embedding"} <= ops, sorted(ops)
        tokens = {key[1][2] for key in rep.rows if key[0] == "attention"}
        assert {hw[0] * hw[1] // 4, hw[0] * hw[1] // 16} <= tokens, sorted(tokens)
