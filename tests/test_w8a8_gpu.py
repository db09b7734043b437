"""GPU tests of the W8A8 path on an H100.

int8 convolution.  int32 accumulation is exact, so each launch is replayed exactly on the CPU: the integer product in
float64 (|q| <= 127 over K <= 23040 terms stays below 2^53), then the epilogue in float64 from the kernel's own
fp32 view of it -- fp32(acc) * col_scale + bias + residual.  The fp16 output must be within one fp16 ulp of that value
plus 2^-20 * B, B = col_scale * (|A| . |W|^T) + |bias| + |residual|: the epilogue's product and two additions are fp32
(2^-24 relative each), and split-K converts and scales each split's partial sum separately, so a partial may be as
large as col_scale * (|A| . |W|^T) even where the whole sum is small.  That matters only where the terms cancel to a
result far below them (measured: errors up to 2e-6 at |out| ~ 1e-4).

Operand producers.  group_norm_s8 / upsample2x_s8 against float64: |q - q64| <= 1 everywhere, and q == q64 wherever
y64 * inv_scale is more than 1e-3 from a half-integer (the fp32 GroupNorm and SiLU may move a value across a rounding
boundary only when it lies that close to one)."""
import os
import sys

import numpy as np
import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import w8a8_oracle as WQ  # noqa: E402

pytestmark = pytest.mark.gpu
WIDTHS = (256, 192, 160, 128, 96, 64, 32, 16)


def _f16_ulp(v):
    a = np.abs(v.astype(np.float64))
    e = np.floor(np.log2(np.maximum(a, 2.0 ** -14)))
    return 2.0 ** (e - 10)


def _conv_ref(x8, w8, col_scale, bias, bias_rows, residual, rows):
    """float64 reference of output rows `rows` of one int8 launch (NHWC x8 [n, h, w, c], w8 [N, 9c] OHWI, bias [N] or
    per-image rows [n, >= N]); returns (ref, B) [len(rows), N] with B the magnitude bound of the docstring."""
    n, h, w, c = x8.shape
    cout = w8.shape[0]
    assert bias is None or bias.dim() == 1 or bias_rows == h * w  # per-image bias rows
    xp = torch.nn.functional.pad(x8.permute(0, 3, 1, 2).to(torch.int16), (1, 1, 1, 1))  # [n, c, h + 2, w + 2]
    img, rem = rows // (h * w), rows % (h * w)
    y, x = rem // w, rem % w
    a = torch.cat([xp[img, :, y + dy, x + dx] for dy in range(3) for dx in range(3)], 1).double()  # tap-major = OHWI
    wd = w8.double()
    acc = a @ wd.t()
    out = acc.float().double() * col_scale.double()[None, :]  # the kernel converts the exact int32 sum to fp32
    mag = (a.abs() @ wd.abs().t()) * col_scale.double()[None, :]
    if bias is not None:
        b = bias.double()[img, :cout] if bias.dim() == 2 else bias.double()[None, :]
        out, mag = out + b, mag + b.abs()
    if residual is not None:
        r = residual.reshape(n * h * w, -1)[rows].double()
        out, mag = out + r, mag + r.abs()
    return out, mag


def _check_launch(x8, w8, cs, bias, bias_rows, residual, out, what, max_rows=4096):
    """Checks a random sample of max_rows output rows plus the last 128 (the tail tile) -- every row when there are few."""
    m = out.numel() // out.shape[-1]
    if m <= max_rows + 128:
        rows = torch.arange(m)
    else:
        pick = torch.randperm(m - 128, generator=torch.Generator().manual_seed(0))[:max_rows]
        rows = torch.cat([pick.sort().values, torch.arange(m - 128, m)])
    ref, mag = _conv_ref(x8.cpu(), w8.cpu(), cs.cpu(), None if bias is None else bias.cpu(), bias_rows,
                         None if residual is None else residual.cpu(), rows)
    ref, mag = ref.numpy(), mag.numpy()
    got = out.reshape(m, -1)[rows.to(out.device)].cpu().double().numpy()
    err = np.abs(got - ref)
    bad = err > _f16_ulp(ref) + 2.0 ** -20 * mag
    idx = np.argwhere(bad)[:6]
    detail = ", ".join(f"[{int(rows[i])},{j}] ref={ref[i, j]!r} got={got[i, j]!r}" for i, j in idx)
    assert not bad.any(), f"{what}: {bad.sum()} of {bad.size} outputs off by more than one fp16 ulp: {detail}"


def _rand_case(g, n, h, w, c, cout, dev):
    x8 = torch.randint(-127, 128, (n, h, w, c), generator=g, dtype=torch.int8).to(dev)
    w8 = torch.randint(-127, 128, (cout, 9 * c), generator=g, dtype=torch.int8).to(dev)
    cs = (torch.rand(cout, generator=g) * 1e-4 + 1e-6).to(dev)
    return x8, w8, cs


CASES = [  # (n, h, w, c, cout, bias kind, residual)
    (2, 16, 16, 320, 320, "rows", False),
    (2, 8, 8, 1280, 1280, "vec", True),
    (2, 32, 32, 640, 640, "vec", True),
    (2, 12, 20, 48, 96, "rows", True),
    (2, 64, 64, 960, 320, "rows", False),
]


@pytest.mark.parametrize("case", CASES)
def test_conv3x3_s8_planned_launch_is_exact(cuda_lib, case):
    from b200sd import lib as L

    n, h, w, c, cout, bk, res = case
    dev = torch.device("cuda:0")
    g = torch.Generator().manual_seed(CASES.index(case))
    x8, w8, cs = _rand_case(g, n, h, w, c, cout, dev)
    bias = (torch.randn(n, cout, generator=g) if bk == "rows" else torch.randn(cout, generator=g)).to(dev)
    residual = torch.randn(n, h, w, cout, generator=g).half().to(dev) if res else None
    out = L.conv3x3_s8(x8, w8, cs, bias, residual, bias_rows=h * w if bk == "rows" else 0)
    out2 = L.conv3x3_s8(x8, w8, cs, bias, residual, bias_rows=h * w if bk == "rows" else 0)
    torch.cuda.synchronize()
    assert torch.equal(out, out2)
    _check_launch(x8, w8, cs, bias, h * w if bk == "rows" else 0, residual, out, str(case))


@pytest.mark.parametrize("bn", WIDTHS)
@pytest.mark.parametrize("split,cluster", [(1, "1"), (3, "0"), (2, "1"), (4, "1")])
def test_conv3x3_s8_forced_plans_are_exact(cuda_lib, monkeypatch, bn, split, cluster):
    from b200sd import lib as L

    monkeypatch.setenv("B200SD_CLUSTER_SPLITK", cluster)
    dev = torch.device("cuda:0")
    g = torch.Generator().manual_seed(bn * 10 + split)
    n, h, w, c, cout = 2, 16, 8, 256, 256
    x8, w8, cs = _rand_case(g, n, h, w, c, cout, dev)
    bias = torch.randn(n, cout, generator=g).to(dev)
    residual = torch.randn(n, h, w, cout, generator=g).half().to(dev)
    args = L.gemm_args(1, x8, w8, torch.empty(1, dtype=torch.float16), n=cout, n_img=n, h=h, w=w, bias_rows=h * w,
                       split_k=split, block_n=bn)
    args.bias, args.residual = 1, 1
    plan = L.plan_ex_s8(args)
    assert plan[0] == bn
    out = L.conv3x3_s8(x8, w8, cs, bias, residual, bias_rows=h * w, split_k=split, block_n=bn)
    torch.cuda.synchronize()
    _check_launch(x8, w8, cs, bias, h * w, residual, out, f"bn={bn} split={split} cluster={cluster}")


def _gn_ref(x, x1, gamma, beta, groups, eps, silu):
    xx = x.double() if x1 is None else torch.cat([x.double(), x1.double()], -1)
    n, h, w, c = xx.shape
    v = xx.reshape(n, h * w, groups, c // groups)
    mu = v.mean((1, 3), keepdim=True)
    var = ((v - mu) ** 2).mean((1, 3), keepdim=True)
    y = ((v - mu) / torch.sqrt(var + eps)).reshape(n, h, w, c) * gamma.double() + beta.double()
    return y * torch.sigmoid(y) if silu else y


def _check_q(q, y64, inv, what):
    t = y64 * inv
    q64 = torch.clamp(torch.round(t), -127, 127)
    d = (q.cpu().double() - q64).abs()
    assert d.max() <= 1, f"{what}: |q - q64| = {d.max()}"
    near = ((t - torch.floor(t) - 0.5).abs() <= 1e-3) & (t.abs() < 127.5)
    assert not (d[~near] > 0).any(), f"{what}: {int((d[~near] > 0).sum())} values differ away from a rounding boundary"


# (n, hw, c0, c1): the cluster kernel and, at 128^2 with 960 channels (SDXL's up_blocks.2.resnets.0), the two-kernel path
@pytest.mark.parametrize("shape", [(2, 16, 320, 0), (2, 32, 640, 320), (2, 8, 1280, 1280), (2, 128, 640, 320)])
def test_group_norm_s8_matches_fp64(cuda_lib, shape):
    from b200sd import lib as L

    n, hw, c0, c1 = shape
    g = torch.Generator().manual_seed(hw + c0)
    x = (torch.randn(n, hw, hw, c0, generator=g) * 2 + 0.5).half()
    x1 = (torch.randn(n, hw, hw, c1, generator=g) * 0.5).half() if c1 else None
    gamma = torch.rand(c0 + c1, generator=g) + 0.5
    beta = torch.randn(c0 + c1, generator=g) * 0.2
    y64 = _gn_ref(x, x1, gamma, beta, 32, 1e-5, True)
    inv = 127.0 / float(y64.abs().max()) * 1.3  # some values saturate
    q = L.group_norm_s8(x.cuda(), gamma.cuda(), beta.cuda(), 32, 1e-5, inv, silu=True,
                        x1=None if x1 is None else x1.cuda())
    torch.cuda.synchronize()
    _check_q(q, y64, inv, str(shape))


def test_upsample2x_s8_matches_fp64(cuda_lib):
    from b200sd import lib as L

    g = torch.Generator().manual_seed(9)
    x = (torch.randn(2, 16, 24, 640, generator=g) * 3).half()
    inv = 127.0 / 8.0
    q = L.upsample2x_s8(x.cuda(), inv)
    torch.cuda.synchronize()
    y64 = x.double().repeat_interleave(2, 1).repeat_interleave(2, 2)
    _check_q(q, y64, inv, "upsample2x_s8")


def test_absmax_probe(cuda_lib):
    from b200sd import lib as L

    x = torch.randn(3, 17, 19, 64).half().cuda()
    slot = torch.zeros(1, device="cuda")
    L.absmax(x, slot)
    L.absmax(x * 0.5, slot)
    assert float(slot) == float(x.abs().max().float())


# ---------------------------------------------------------------------------------------------------------------------
# UNet
# ---------------------------------------------------------------------------------------------------------------------
def _unet_inputs(cfg, batch, hw, seed=2):
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(batch, 4, hw, hw, generator=g)
    ctx = torch.randn(batch, cfg["cross_attention_dim"], 1, 77, generator=g)
    t = torch.full((batch,), 501.0)
    return x, t, ctx


def _full_recipe(sd, cfg, x, t, ctx):
    """Scales of every quantizable layer from an oracle calibration pass on the same inputs."""
    from b200sd import quantization as Q
    from oracle import restated as R  # noqa: F401

    layers = Q.quantizable_layers(cfg)
    with torch.no_grad():
        amax = WQ.calibrate(sd, cfg, x, t, ctx, set(layers))
    return Q.W8A8Recipe.from_amax(amax, cfg)


def test_unet_empty_recipe_is_bit_identical(cuda_lib):
    from b200sd import config as C
    from b200sd import quantization as Q
    from b200sd.model import UNetModel

    cfg = C.TINY_UNET
    sd = C.random_state_dict(C.unet_param_shapes(cfg), seed=1)
    x, t, ctx = _unet_inputs(cfg, 2, 16)
    kw = dict(sample=x.half().numpy(), timestep=t.half().numpy(), encoder_hidden_states=ctx.half().numpy())
    a = UNetModel(cfg, sd, batch=2, height=16, width=16)(**kw)["noise_pred"]
    b = UNetModel(cfg, sd, batch=2, height=16, width=16, quantization=Q.W8A8Recipe({}, Q.architecture(cfg)))(**kw)["noise_pred"]
    assert np.array_equal(a, b)


@pytest.mark.parametrize("model", ["tiny", "sd21"])
def test_unet_full_recipe_tracks_the_fake_quant_oracle(cuda_lib, model):
    """rms(engine - oracle_q) <= 1.5 * rms(oracle_q - oracle_fp32).  The engine stores activations in fp16, so an
    activation close to a rounding boundary of its int8 grid can land one quantum away from the oracle's; those flips
    are the same size as the quantization error itself.  The bound 0.5 first chosen does not hold: on an H100 the
    ratio measured 1.09 (tiny config) and 1.07 (SD-2.1-base, 32^2 latents), so 1.5 is a bound set from that
    measurement with some margin, not derived."""
    from b200sd import config as C
    from b200sd.model import UNetModel
    from oracle import restated as R

    cfg, hw = (C.TINY_UNET, 16) if model == "tiny" else (C.SD21_BASE_UNET, 32)
    sd = {k: v.half().float() for k, v in C.random_state_dict(C.unet_param_shapes(cfg), seed=3).items()}
    x, t, ctx = _unet_inputs(cfg, 2, hw)
    x, ctx = x.half().float(), ctx.half().float()
    recipe = _full_recipe(sd, cfg, x, t, ctx)
    with torch.no_grad():
        ref32 = R.unet_forward(sd, cfg, x, t, ctx)
        refq = WQ.unet_forward_q(sd, cfg, x, t, ctx, recipe.scales)
    u = UNetModel(cfg, {k: v.half() for k, v in sd.items()}, batch=2, height=hw, width=hw, quantization=recipe)
    got = torch.from_numpy(u(sample=x.half().numpy(), timestep=t.half().numpy(),
                             encoder_hidden_states=ctx.half().numpy())["noise_pred"]).double()
    rms = lambda d: float(d.double().pow(2).mean().sqrt())  # noqa: E731
    e_engine, e_quant = rms(got - refq), rms(refq - ref32)
    assert e_quant > 0 and e_engine <= 1.5 * e_quant, f"{model}: engine-vs-q {e_engine:.4g}, q-vs-fp32 {e_quant:.4g}"


# ---------------------------------------------------------------------------------------------------------------------
# pipeline
# ---------------------------------------------------------------------------------------------------------------------
def test_pipeline_w8a8_calibration_loop_graph_and_determinism(cuda_lib, tmp_path):
    from b200sd import config as C
    from b200sd import quantization as Q
    from b200sd.model import UNetModel
    from b200sd.pipeline import B200StableDiffusionPipeline as P

    pipe = P.from_random_init("tiny", images_per_call=1, seed=0, height=64, width=64)
    recipe = pipe.calibrate_unet(["a photo of a cat"], num_inference_steps=4, guidance_scale=7.5, seed=1)
    assert len(recipe) == len(Q.quantizable_layers(C.TINY_UNET))
    assert all(s > 0 for s in recipe.scales.values())
    path = tmp_path / "recipe.json"
    recipe.save(path)
    u = pipe.unet
    usd = C.random_state_dict(C.unet_param_shapes(C.TINY_UNET), seed=0, dtype=torch.float16)  # from_random_init's
    pipe.unet = UNetModel(C.TINY_UNET, usd, batch=u.batch, height=u.h, width=u.w, quantization=str(path))
    pipe._loop_graphs = {}
    lat = torch.from_numpy(np.random.RandomState(0).randn(1, 4, u.h, u.w).astype(np.float32))
    emb = torch.from_numpy(np.random.RandomState(1).randn(2, C.TINY_UNET["cross_attention_dim"], 1, 77).astype(np.float16))
    a = pipe.denoise(emb, lat, 4, 7.5).clone()
    b = pipe.denoise(emb, lat, 4, 7.5).clone()
    c = pipe.denoise(emb, lat, 4, 7.5, record=[]).clone()  # step by step
    assert torch.isfinite(a).all()
    assert torch.equal(a, b), "two runs of the loop graph differ"
    assert torch.equal(a, c), "loop graph and step-by-step path differ"


# ---------------------------------------------------------------------------------------------------------------------
# every int8 launch of the W8A8 models
# ---------------------------------------------------------------------------------------------------------------------
_FUSION_ENV = ("B200SD_FUSED", "B200SD_HALO_TMA", "B200SD_FOLD_SC", "B200SD_CLUSTER_SPLITK", "B200SD_SMEM_KB",
               "B200SD_STAGED", "B200SD_TILED_W")


@pytest.mark.parametrize("name", ["sd21_b2", "sd15_b2", "sdxl_1024_b2", "sd15_512x768_b2", "sdxl_768x1344_b2"])
def test_every_int8_launch_of_the_w8a8_models_is_exact(cuda_lib, monkeypatch, name):
    """W8A8 SD-2.1-base and SD-1.5 at 512^2, SDXL at 1024^2, and SD-1.5 at 512x768 and SDXL at 768x1344 on non-square
    maps (random init, batch 2), every eligible layer quantized
    with scales from a calibration pass of the fp16 engine on the same inputs.  Every conv3x3_s8 launch of one forward
    is recorded and replayed exactly on the CPU (a sample of 1024 rows plus the tail tile per launch), with the plan the
    planner picks for it."""
    import model_cases as MC
    from b200sd import config as C
    from b200sd import lib as L
    from b200sd import quantization as Q
    from b200sd.model import UNetModel

    for k in _FUSION_ENV:
        monkeypatch.delenv(k, raising=False)
    m = MC.build(name)  # fp16, random init seed 5
    cfg, batch, lat_h, lat_w = dict(m.engine.cfg), m.batch, m.h, m.w
    inputs = MC.model_inputs(m, seed=1)
    slots = m.engine.set_calibration(True)
    m(**inputs)
    recipe = Q.W8A8Recipe.from_amax({k: float(v) for k, v in slots.items()}, cfg)
    assert len(recipe) == len(Q.quantizable_layers(cfg))
    del m, slots
    torch.cuda.empty_cache()
    sd = C.random_state_dict(C.unet_param_shapes(cfg), seed=5, dtype=torch.float16)
    qm = UNetModel(cfg, sd, batch=batch, height=lat_h, width=lat_w, use_cuda_graph=False, quantization=recipe)
    del sd
    calls = []
    orig = L.conv3x3_s8

    def record(x, wgt, col_scale, bias=None, residual=None, *, bias_rows=0, bias_stride=0, split_k=0, block_n=0, out=None):
        o = orig(x, wgt, col_scale, bias, residual, bias_rows=bias_rows, bias_stride=bias_stride, split_k=split_k,
                 block_n=block_n, out=out)
        calls.append((x, wgt, col_scale, bias, bias_rows, residual, o))
        return o

    monkeypatch.setattr(L, "conv3x3_s8", record)
    out = qm(**inputs)["noise_pred"]
    torch.cuda.synchronize()
    assert np.isfinite(out).all()
    assert len(calls) == len(recipe), (len(calls), len(recipe))
    for layer, (x8, w8, cs, bias, bias_rows, residual, o) in zip(recipe.scales, calls):
        n, h, w, c = x8.shape
        plan = L.describe_plan_s8(w8.shape[0], c, n, h, w, has_bias=bias is not None, has_residual=residual is not None,
                                  bias_rows=bias_rows)
        _check_launch(x8, w8, cs, bias, bias_rows, residual, o, f"{name} {layer} ({plan})", max_rows=1024)


def test_from_pretrained_with_a_saved_recipe(cuda_lib, tmp_path):
    """calibrate_unet -> saved recipe -> from_pretrained(model dir, unet_quantization=path) generates images."""
    import test_factory_gpu as TF
    from b200sd import config as C
    from b200sd.pipeline import B200StableDiffusionPipeline as P

    TF._model_dir(tmp_path, C.TINY_UNET, seed=11)
    pipe = P.from_pretrained(str(tmp_path), height=64, width=64)
    recipe = pipe.calibrate_unet(["a red cube"], num_inference_steps=3, seed=2)
    path = tmp_path / "w8a8.json"
    recipe.save(path)
    qpipe = P.from_pretrained(str(tmp_path), height=64, width=64, unet_quantization=str(path))
    assert len(qpipe.unet.engine.q) == len(recipe)
    kw = dict(height=64, width=64, num_inference_steps=3, guidance_scale=5.0, output_type="np", seed=7)
    img = qpipe("a red cube", **kw).images
    ref = pipe("a red cube", **kw).images
    assert img.shape == ref.shape == (1, 64, 64, 3) and np.isfinite(img).all()
    assert not np.array_equal(img, ref)  # the quantized layers did run


def test_refiner_stays_fp16_beside_a_w8a8_base(cuda_lib):
    """An SDXL pipeline with a W8A8 base UNet keeps its refiner fp16: with the hand-off at step 0 (the refiner runs
    every step) the latents are bit-identical to the same pipeline with the fp16 base."""
    import model_cases as MC
    from b200sd import config as C
    from b200sd import quantization as Q
    from b200sd.model import UNetModel
    from b200sd.pipeline import B200StableDiffusionPipeline as P
    from b200sd.vae import VAEDecoderModel

    bcfg = C.TINY_XL_UNET
    rcfg = dict(bcfg, projection_class_embeddings_input_dim=64 + 5 * 32, num_time_ids=5)
    bsd = C.random_state_dict(C.unet_param_shapes(bcfg), seed=21, dtype=torch.float16)
    rsd = C.random_state_dict(C.unet_param_shapes(rcfg), seed=22, dtype=torch.float16)
    vsd = C.random_state_dict(C.vae_decoder_param_shapes(C.TINY_VAE), seed=23, dtype=torch.float16)
    base16 = UNetModel(bcfg, bsd, batch=2, height=16, width=16, use_cuda_graph=False)
    slots = base16.engine.set_calibration(True)
    base16(**MC.model_inputs(base16, seed=4))
    recipe = Q.W8A8Recipe.from_amax({k: float(v) for k, v in slots.items()}, bcfg)
    base16.engine.set_calibration(False)
    base16.use_cuda_graph = True  # the refiner hand-off runs in the pipeline's loop graph
    base8 = UNetModel(bcfg, bsd, batch=2, height=16, width=16, quantization=recipe)
    g = torch.Generator().manual_seed(3)
    emb, pooled = torch.randn(2, 96, 1, 77, generator=g).half(), torch.randn(2, 64, generator=g)
    remb, rpooled = torch.randn(2, 96, 1, 77, generator=g).half(), torch.randn(2, 64, generator=g)
    lat0 = torch.randn(1, 4, 16, 16, generator=g)
    tid = torch.tensor([[64.0, 64.0, 0.0, 0.0, 64.0, 64.0]] * 2)
    rtid = torch.tensor([[64.0, 64.0, 0.0, 0.0, 2.5], [64.0, 64.0, 0.0, 0.0, 6.0]])
    outs = []
    for base in (base16, base8):
        refiner = UNetModel(rcfg, rsd, batch=2, height=16, width=16)
        assert refiner.engine.recipe is None and not refiner.engine.q
        pipe = P(base, VAEDecoderModel(C.TINY_VAE, vsd, batch=1, height=16, width=16), scheduler="DDIM", xl=True,
                 unet_refiner=refiner)
        ref_in = {"encoder_hidden_states": remb, "time_ids": rtid, "text_embeds": rpooled}
        outs.append(pipe.denoise(emb, lat0, 4, 4.0, time_ids=tid, text_embeds=pooled, refiner=ref_in,
                                 refiner_start=0.0).cpu().clone())
        # with the hand-off late, the base (W8A8 or fp16) runs first
        outs.append(pipe.denoise(emb, lat0, 4, 4.0, time_ids=tid, text_embeds=pooled, refiner=ref_in,
                                 refiner_start=0.5).cpu().clone())
    assert torch.equal(outs[0], outs[2])
    assert torch.isfinite(outs[3]).all() and not torch.equal(outs[1], outs[3])


def test_calibration_rejects_the_opt_in_fusion_levels(cuda_lib, monkeypatch):
    from b200sd import config as C
    from b200sd.unet import UNetEngine

    monkeypatch.setenv("B200SD_FUSED", "1")
    sd = C.random_state_dict(C.unet_param_shapes(C.TINY_UNET), seed=1, dtype=torch.float16)
    eng = UNetEngine(C.TINY_UNET, sd, "cuda:0")
    with pytest.raises(ValueError, match="B200SD_FUSED"):
        eng.set_calibration(True)
