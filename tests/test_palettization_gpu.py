"""Palettized weights on the GPU: every b200sd_gemm_lut launch is bit-identical to the fp16 kernel on the decoded
weights, and so is the whole palettized UNet to the fp16 UNet built from palettization.decoded_state_dict."""
import gc

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

WIDTHS = [256, 192, 160, 128, 96, 64, 32]


def _pw(w2d, nbits, dev, kscale=None, segments=None):
    from b200sd import palettization as Pz

    segments = segments or [(w2d, nbits)]
    fits = [Pz.fit_palette(w.to(dev), n) + (n,) for w, n in segments]
    pw = Pz.palettized(fits, kscale)
    return pw, pw.decoded()


@pytest.mark.parametrize("nbits", [1, 2, 4, 6, 8])
def test_linear_launches_are_exact(cuda_lib, nbits):
    from b200sd import lib as L

    dev = torch.device("cuda:0")
    g = torch.Generator().manual_seed(nbits)
    m, c = 512, 640
    x = torch.randn(m, c, generator=g).half().to(dev)
    res = torch.randn(m, c, generator=g).half().to(dev)
    bias = torch.randn(c, generator=g).to(dev)
    pw, wd = _pw(torch.randn(c, c, generator=g) * 0.05, nbits, dev)
    rs_a, rs_b = {}, {}
    a = L.linear(x, pw, bias, res, rowstats=rs_a)
    b = L.linear(x, wd, bias, res, static_w=True, rowstats=rs_b)
    assert torch.equal(a, b)
    assert torch.equal(rs_a["rows"], rs_b["rows"])
    # plain, and a ragged N (rows past N decode to zero)
    pw2, wd2 = _pw(torch.randn(336, c, generator=g) * 0.05, nbits, dev)
    assert torch.equal(L.linear(x, pw2, None), L.linear(x, wd2, None, static_w=True))
    # LayerNorm-folded, segmented qkv with mixed widths: gamma applied in the decode
    gamma = (torch.rand(c, generator=g) + 0.5).to(dev)
    segs = [(torch.randn(c, c, generator=g) * 0.05, n) for n in (nbits, 4, 2)]
    pw3, wd3 = _pw(None, None, dev, kscale=gamma, segments=segs)
    assert pw3.nbits == max(nbits, 4)
    stat = torch.stack([torch.randn(2, m, generator=g) * 10, (1 + torch.rand(2, m, generator=g)) * c], -1).to(dev)
    ln = dict(stat=stat, parts=2, wg=wd3.float().sum(1).contiguous(), eps=1e-5)
    assert torch.equal(L.linear(x, pw3, bias.repeat(3), ln=ln), L.linear(x, wd3, bias.repeat(3), ln=ln, static_w=True))
    # GEGLU with the fold
    pw4, wd4 = _pw(torch.randn(4 * c, c, generator=g) * 0.05, nbits, dev, kscale=gamma)
    ln4 = dict(stat=stat, parts=2, wg=wd4.float().sum(1).contiguous(), eps=1e-5)
    b4 = torch.randn(4 * c, generator=g).to(dev)
    assert torch.equal(L.linear(x, pw4, b4, geglu=True, ln=ln4), L.linear(x, wd4, b4, geglu=True, ln=ln4, static_w=True))


@pytest.mark.parametrize("nbits", [1, 2, 4, 6, 8])
@pytest.mark.parametrize("shape", [(2, 16, 16, 128, 64, 128, 1), (2, 8, 8, 1280, 0, 1280, 1), (2, 32, 32, 320, 0, 320, 2)])
def test_conv_launches_are_exact(cuda_lib, nbits, shape):
    from b200sd import lib as L

    dev = torch.device("cuda:0")
    n, h, w, c0, c1, co, stride = shape
    g = torch.Generator().manual_seed(nbits + c0)
    x = torch.randn(n, h, w, c0, generator=g).half().to(dev)
    x1 = torch.randn(n, h, w, c1, generator=g).half().to(dev) if c1 else None
    pw, wd = _pw(torch.randn(co, 9 * (c0 + c1), generator=g) * 0.02, nbits, dev)
    if stride == 1:
        bias = torch.randn(n, co, generator=g).to(dev)
        res = torch.randn(n, h, w, co, generator=g).half().to(dev)
        kw = dict(bias_rows=h * w)
        a = L.conv3x3(x, pw, bias, res, x1=x1, **kw)
        b = L.conv3x3(x, wd, bias, res, x1=x1, **kw)
    else:
        bias = torch.randn(co, generator=g).to(dev)
        a = L.conv3x3(x, pw, bias, stride=2)
        b = L.conv3x3(x, wd, bias, stride=2)
    assert torch.equal(a, b)


@pytest.mark.parametrize("bn", WIDTHS)
@pytest.mark.parametrize("split,cluster", [(1, "1"), (3, "0"), (2, "1")])
def test_forced_plans_are_exact(cuda_lib, monkeypatch, bn, split, cluster):
    from b200sd import lib as L

    monkeypatch.setenv("B200SD_CLUSTER_SPLITK", cluster)
    dev = torch.device("cuda:0")
    g = torch.Generator().manual_seed(bn * 10 + split)
    n, h, w, c, co = 2, 16, 8, 256, 256
    x = torch.randn(n, h, w, c, generator=g).half().to(dev)
    bias = torch.randn(n, co, generator=g).to(dev)
    res = torch.randn(n, h, w, co, generator=g).half().to(dev)
    pw, wd = _pw(torch.randn(co, 9 * c, generator=g) * 0.02, 4, dev)
    args = L.gemm_args(1, x, pw.packed, torch.empty(1, dtype=torch.float16), n=co, n_img=n, h=h, w=w, bias_rows=h * w,
                       split_k=split, block_n=bn)
    args.bias, args.residual = 1, 1
    desc = L.describe_plan_lut(args, pw)
    assert f"block_n={bn} " in desc, desc
    kw = dict(bias_rows=h * w, split_k=split, block_n=bn)
    assert torch.equal(L.conv3x3(x, pw, bias, res, **kw), L.conv3x3(x, wd, bias, res, static_w=False, **kw))


def _inputs(cfg, batch, hw, seed=2):
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(batch, 4, hw, hw, generator=g)
    ctx = torch.randn(batch, cfg["cross_attention_dim"], 1, 77, generator=g)
    t = torch.full((batch,), 501.0)
    return dict(sample=x.half().numpy(), timestep=t.half().numpy(), encoder_hidden_states=ctx.half().numpy())


def _mixed(cfg):
    from b200sd import palettization as Pz

    layers = list(Pz.palettizable_layers(cfg))
    return {name: (1, 2, 4, 6, 8, 16)[i % 6] for i, name in enumerate(layers)}


@pytest.mark.parametrize("model,recipe", [("tiny", 4), ("tiny", "mixed"), ("sd21", 4), ("sd21", "mixed")])
def test_unet_matches_the_decoded_fp16_unet(cuda_lib, monkeypatch, model, recipe):
    """A palettized conv2 does not take the folded ResNet shortcut, so both engines run the shortcut as its own launch
    (B200SD_FOLD_SC=0) to share one launch sequence."""
    from b200sd import config as C
    from b200sd import palettization as Pz
    from b200sd.model import UNetModel

    cfg = C.TINY_UNET if model == "tiny" else C.SD21_BASE_UNET
    hw = 16 if model == "tiny" else 32
    sd = C.random_state_dict(C.unet_param_shapes(cfg), seed=1, dtype=torch.float16)
    rec = _mixed(cfg) if recipe == "mixed" else recipe
    dec = Pz.decoded_state_dict(sd, rec, cfg)
    kw = _inputs(cfg, 2, hw)
    monkeypatch.setenv("B200SD_FOLD_SC", "0")
    for graph in (False, True):
        pal = UNetModel(cfg, sd, batch=2, height=hw, width=hw, palettization=rec, use_cuda_graph=graph)
        ref = UNetModel(cfg, dec, batch=2, height=hw, width=hw, use_cuda_graph=graph)
        a = pal(**kw)["noise_pred"]
        b = ref(**kw)["noise_pred"]
        assert np.isfinite(a).all()
        assert np.array_equal(a, b), f"graph={graph}: max diff {np.abs(a - b).max()}"
        assert pal.engine.weight_bytes < ref.engine.weight_bytes
        del pal, ref


def test_resolution_change_stays_exact(cuda_lib, monkeypatch):
    """An engine built for 16^2 latents runs 24^2 next (other tile plans, the same packed indices)."""
    from b200sd import config as C
    from b200sd import lib as L
    from b200sd import palettization as Pz
    from b200sd.model import UNetModel

    cfg = C.TINY_UNET
    sd = C.random_state_dict(C.unet_param_shapes(cfg), seed=3, dtype=torch.float16)
    monkeypatch.setenv("B200SD_FOLD_SC", "0")
    pal = UNetModel(cfg, sd, batch=2, height=16, width=16, palettization=4, use_cuda_graph=False)
    ref = UNetModel(cfg, Pz.decoded_state_dict(sd, 4, cfg), batch=2, height=16, width=16, use_cuda_graph=False)
    kw = _inputs(cfg, 2, 16)
    assert np.array_equal(pal(**kw)["noise_pred"], ref(**kw)["noise_pred"])
    kw24 = _inputs(cfg, 2, 24)
    x = torch.from_numpy(kw24["sample"]).float()

    def run(engine):
        xs = L.nchw_to_nhwc(x.cuda(), c_pad=engine.in_pad)
        ctx = L.ctx_to_tokens(torch.from_numpy(kw24["encoder_hidden_states"]).cuda())
        return engine.forward(xs, torch.full((2,), 501.0, device="cuda"), ctx, 77)

    assert torch.equal(run(pal.engine), run(ref.engine))


def _expected_weight_bytes(pal, ref):
    """The palettized engine's resident bytes from the fp16 engine's and the recipe: each palettized launch's fp16
    operand [N, K] replaced by N * row_bytes(K, container bits) packed bytes and the [3][256] fp16 palette table (a
    folded launch's per-k scale is the LayerNorm gamma the engine holds anyway); the unfolded twins of folded launches
    (never run) dropped."""
    from b200sd import palettization as Pz

    total = ref.weight_bytes
    def visit(p, r):
        nonlocal total
        for k, v in p.items() if isinstance(p, dict) else enumerate(p):
            if isinstance(v, Pz.PalettizedWeight):
                n, kk = r[k].shape
                bits = max(pal.palettization[name] for name in v.layers)
                total += n * Pz.row_bytes(kk, bits) + 3 * 256 * 2 - r[k].numel() * 2
            elif isinstance(v, (dict, list)):
                visit(v, r[k])
        if isinstance(p, dict):
            for k in set(r) - set(p):
                total -= r[k].numel() * r[k].element_size()
    visit(pal.w, ref.w)
    return total


def test_weight_bytes_and_resident_memory(cuda_lib, monkeypatch):
    """SD-2.1-base at 4 bits: weight_bytes equals the figure computed from the recipe, and the device memory the build
    and first forward add stays within weight_bytes plus the fp16 engine's activation and workspace footprint (a
    surviving fp16 copy of the palettized weights would add about 1.7 GB)."""
    from b200sd import config as C
    from b200sd import lib as L
    from b200sd import palettization as Pz
    from b200sd.model import UNetModel

    cfg = C.SD21_BASE_UNET
    sd = C.random_state_dict(C.unet_param_shapes(cfg), seed=4, dtype=torch.float16)
    monkeypatch.setenv("B200SD_FOLD_SC", "0")
    kw = _inputs(cfg, 2, 32)
    dec = Pz.decoded_state_dict(sd, 4, cfg)
    gc.collect()  # models of earlier tests waiting for the collector must not be freed inside the measured window
    torch.cuda.synchronize()
    m0 = torch.cuda.memory_allocated()
    tiled0 = set(L._tiled_cache)
    ref = UNetModel(cfg, dec, batch=2, height=32, width=32, use_cuda_graph=False)
    b = ref(**kw)["noise_pred"]
    torch.cuda.synchronize()
    tiled = sum(v[2].numel() * v[2].element_size() for k, v in L._tiled_cache.items() if k not in tiled0)
    act_f = torch.cuda.memory_allocated() - m0 - ref.engine.weight_bytes - tiled
    m1 = torch.cuda.memory_allocated()
    pal = UNetModel(cfg, sd, batch=2, height=32, width=32, palettization=4, use_cuda_graph=False)
    a = pal(**kw)["noise_pred"]
    torch.cuda.synchronize()
    grow_p = torch.cuda.memory_allocated() - m1
    assert np.array_equal(a, b)
    assert pal.engine.weight_bytes == _expected_weight_bytes(pal.engine, ref.engine)
    assert pal.engine.weight_bytes < 0.4 * ref.engine.weight_bytes
    assert grow_p <= pal.engine.weight_bytes + max(act_f, 0) + (64 << 20), (grow_p, pal.engine.weight_bytes, act_f)
    once = ("time_embedding.", ".time_emb_proj", ".attn2.to_k", ".attn2.to_v")
    for name, (nominal, stored) in pal.engine.stored_bits().items():
        assert nominal == 4 and stored == (16 if any(o in name for o in once) else 4), (name, stored)


def _record_lut_launches(model):
    """The palettized launches of one eager forward of a 4-bit engine at a shipped model's shapes, one per distinct
    launch signature: (kind, x, weight, positional args, keyword args)."""
    import model_cases as MC
    from b200sd import config as C
    from b200sd import lib as L
    from b200sd import palettization as Pz
    from b200sd.model import UNetModel

    cfg = {"sd21": C.SD21_BASE_UNET, "sd15": C.SD15_UNET, "sdxl": C.SDXL_BASE_UNET}[model[:4]]
    h, w = MC.latent_hw(model)
    sd = C.random_state_dict(C.unet_param_shapes(cfg), seed=5, dtype=torch.float16)
    m = UNetModel(cfg, sd, batch=2, height=h, width=w, palettization=4, use_cuda_graph=False)
    del sd
    calls = {}
    orig = {"linear": L.linear, "conv3x3": L.conv3x3}

    def recorder(kind):
        def rec(x, wgt, *a, **k):
            if isinstance(wgt, Pz.PalettizedWeight):
                key = (kind, tuple(x.shape), wgt.shape, wgt.seg_ends, wgt.kscale is not None, tuple(sorted(k)),
                       tuple(t is not None for t in a), k.get("stride", 1))
                calls.setdefault(key, (kind, x, wgt, a, dict(k)))
            return orig[kind](x, wgt, *a, **k)
        return rec

    L.linear, L.conv3x3 = recorder("linear"), recorder("conv3x3")
    try:
        m(**MC.model_inputs(m, seed=6))
    finally:
        L.linear, L.conv3x3 = orig["linear"], orig["conv3x3"]
    torch.cuda.synchronize()
    return list(calls.values())


@pytest.mark.parametrize("model", ["sd21_b2", "sd15_b2", "sdxl_1024_b2", "sd15_512x768_b2"])
def test_every_palettized_launch_of_the_shipped_models_is_exact(cuda_lib, model):
    """Each distinct palettized launch (ResNet / sampler convolutions, proj_in / proj_out, the folded and segmented
    qkv, q2 and GEGLU launches, attention outputs, ff.net.2) at 1, 2, 4, 6 and 8 bits with random indices and palettes:
    torch.equal to the fp16 kernel on the decoded weights, row statistics included.  SD-1.5 at 512x768 runs every one
    of them on non-square maps."""
    from b200sd import lib as L
    from b200sd import palettization as Pz

    calls = _record_lut_launches(model)
    assert len(calls) >= 10
    g = torch.Generator(device="cuda").manual_seed(7)
    for kind, x, pw, a, k in calls:
        n, kk = pw.shape
        ends = [0, pw.seg_ends[0], pw.seg_ends[1], n]
        for nbits in (1, 2, 4, 6, 8):
            segs = []
            for s in range(3):
                rows = ends[s + 1] - ends[s]
                if rows == 0 and s > 0:
                    continue
                lut = (torch.randn(2 ** nbits, device="cuda", generator=g) * 0.05).half()
                segs.append((lut, torch.randint(0, 2 ** nbits, (rows, kk), device="cuda", generator=g).to(torch.uint8),
                             nbits))
            pwn = Pz.palettized(segs, pw.kscale)
            wd = pwn.decoded()
            fn = getattr(L, kind)
            ka, kb = dict(k), dict(k)
            if "rowstats" in k and k["rowstats"] is not None:
                ka["rowstats"], kb["rowstats"] = {}, {}
            if kind == "linear":
                kb["static_w"] = True
            out_a = fn(x, pwn, *a, **ka)
            out_b = fn(x, wd, *a, **kb)
            what = f"{kind} x={tuple(x.shape)} w={pw.shape} segs={pw.seg_ends} nbits={nbits}"
            assert torch.equal(out_a, out_b), what
            if ka.get("rowstats"):
                assert torch.equal(ka["rowstats"]["rows"], kb["rowstats"]["rows"]), what


def _tiny_pipe(unet, refiner=None):
    from b200sd import config as C
    from b200sd.pipeline import B200StableDiffusionPipeline as P
    from b200sd.vae import VAEDecoderModel

    vsd = C.random_state_dict(C.vae_decoder_param_shapes(C.TINY_VAE), seed=23, dtype=torch.float16)
    return P(unet, VAEDecoderModel(C.TINY_VAE, vsd, batch=1, height=16, width=16), scheduler="DDIM",
             xl=unet.engine.xl, unet_refiner=refiner)


def test_denoise_loop_graph_matches_the_decoded_fp16_unet(cuda_lib, monkeypatch):
    """The whole-loop CUDA graph of denoise() over a mixed-recipe UNet equals the loop over the decoded fp16 UNet."""
    from b200sd import config as C
    from b200sd import palettization as Pz
    from b200sd.model import UNetModel

    cfg = C.TINY_UNET
    monkeypatch.setenv("B200SD_FOLD_SC", "0")
    sd = C.random_state_dict(C.unet_param_shapes(cfg), seed=8, dtype=torch.float16)
    rec = _mixed(cfg)
    g = torch.Generator().manual_seed(3)
    emb = torch.randn(2, cfg["cross_attention_dim"], 1, 77, generator=g).half()
    lat = torch.randn(1, 4, 16, 16, generator=g)
    outs = []
    for unet in (UNetModel(cfg, sd, batch=2, height=16, width=16, palettization=rec),
                 UNetModel(cfg, Pz.decoded_state_dict(sd, rec, cfg), batch=2, height=16, width=16)):
        pipe = _tiny_pipe(unet)
        outs.append(pipe.denoise(emb, lat, 4, 7.5).cpu().clone())
        outs.append(pipe.denoise(emb, lat, 4, 7.5).cpu().clone())
    assert torch.isfinite(outs[0]).all()
    assert torch.equal(outs[0], outs[1]) and torch.equal(outs[0], outs[2]) and torch.equal(outs[2], outs[3])


def test_refiner_stays_fp16_beside_a_palettized_base(cuda_lib):
    """An SDXL pipeline with a palettized base keeps its refiner fp16: with the hand-off at step 0 (the refiner runs
    every step) the latents are bit-identical to the same pipeline with the fp16 base."""
    from b200sd import config as C
    from b200sd.model import UNetModel

    bcfg = C.TINY_XL_UNET
    rcfg = dict(bcfg, projection_class_embeddings_input_dim=64 + 5 * 32, num_time_ids=5)
    bsd = C.random_state_dict(C.unet_param_shapes(bcfg), seed=21, dtype=torch.float16)
    rsd = C.random_state_dict(C.unet_param_shapes(rcfg), seed=22, dtype=torch.float16)
    g = torch.Generator().manual_seed(3)
    emb, pooled = torch.randn(2, 96, 1, 77, generator=g).half(), torch.randn(2, 64, generator=g)
    remb, rpooled = torch.randn(2, 96, 1, 77, generator=g).half(), torch.randn(2, 64, generator=g)
    lat0 = torch.randn(1, 4, 16, 16, generator=g)
    tid = torch.tensor([[64.0, 64.0, 0.0, 0.0, 64.0, 64.0]] * 2)
    rtid = torch.tensor([[64.0, 64.0, 0.0, 0.0, 2.5], [64.0, 64.0, 0.0, 0.0, 6.0]])
    outs = []
    for pal in (None, 4):
        base = UNetModel(bcfg, bsd, batch=2, height=16, width=16, palettization=pal)
        refiner = UNetModel(rcfg, rsd, batch=2, height=16, width=16)
        assert refiner.engine.palettization is None
        pipe = _tiny_pipe(base, refiner)
        ref_in = {"encoder_hidden_states": remb, "time_ids": rtid, "text_embeds": rpooled}
        outs.append(pipe.denoise(emb, lat0, 4, 4.0, time_ids=tid, text_embeds=pooled, refiner=ref_in,
                                 refiner_start=0.0).cpu().clone())
        outs.append(pipe.denoise(emb, lat0, 4, 4.0, time_ids=tid, text_embeds=pooled, refiner=ref_in,
                                 refiner_start=0.5).cpu().clone())
    assert torch.equal(outs[0], outs[2])
    assert torch.isfinite(outs[3]).all() and not torch.equal(outs[1], outs[3])


def test_rejected_combinations(cuda_lib, monkeypatch):
    from b200sd import config as C
    from b200sd import lib as L
    from b200sd import quantization as Q
    from b200sd.unet import UNetEngine

    cfg = C.TINY_UNET
    sd = C.random_state_dict(C.unet_param_shapes(cfg), seed=1, dtype=torch.float16)
    with pytest.raises(ValueError, match="W8A8"):
        UNetEngine(cfg, sd, "cuda:0", quantization=Q.W8A8Recipe({}, Q.architecture(cfg)), palettization=4)
    monkeypatch.setenv("B200SD_FUSED", "1")
    with pytest.raises(ValueError, match="B200SD_FUSED"):
        UNetEngine(cfg, sd, "cuda:0", palettization=4)
    monkeypatch.setenv("B200SD_FUSED", "ln")
    monkeypatch.setenv("B200SD_HALO_TMA", "1024")
    with pytest.raises(ValueError, match="HALO_TMA"):
        UNetEngine(cfg, sd, "cuda:0", palettization=4)
    monkeypatch.delenv("B200SD_HALO_TMA")
    monkeypatch.setenv("B200SD_STAGED", "1")
    with pytest.raises(ValueError, match="B200SD_STAGED"):
        UNetEngine(cfg, sd, "cuda:0", palettization=4)
    monkeypatch.delenv("B200SD_STAGED")
    monkeypatch.setattr(L, "TILED_WEIGHTS", False)
    with pytest.raises(ValueError, match="B200SD_TILED_W"):
        UNetEngine(cfg, sd, "cuda:0", palettization=4)


def test_from_pretrained_with_a_recipe_json(cuda_lib, tmp_path):
    import json

    import test_factory_gpu as TF
    from b200sd import config as C
    from b200sd import palettization as Pz
    from b200sd.pipeline import B200StableDiffusionPipeline as P

    TF._model_dir(tmp_path, C.TINY_UNET, seed=11)
    rec = {k: 4 for k in Pz.palettizable_layers(C.TINY_UNET)}
    path = tmp_path / "recipes.json"
    path.write_text(json.dumps({"model_version": "tiny", "baselines": {}, "recipes": {"recipe_4.00_bit_mixedpalette": rec}}))
    pipe = P.from_pretrained(str(tmp_path), height=64, width=64,
                             unet_palettization=(str(path), "recipe_4.00_bit_mixedpalette"))
    assert pipe.unet.engine.palettization == rec
    kw = dict(height=64, width=64, num_inference_steps=3, guidance_scale=5.0, output_type="np", seed=7)
    img = pipe("a red cube", **kw).images
    assert img.shape == (1, 64, 64, 3) and np.isfinite(img).all()
