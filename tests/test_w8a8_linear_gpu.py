"""GPU tests of the W8A8 transformer linears on an H100.

int8 linear.  As for the int8 convolution (test_w8a8_gpu.py), int32 accumulation is exact, so each launch is replayed
on the CPU in float64 from the kernel's fp32 view of the integer sum: fp32(acc) * col_scale + bias (+ residual).  An fp16
output must be within one fp16 ulp of that plus 2^-20 * B, B the magnitude of the terms.  GEGLU multiplies the value
column by gelu of the gate column: the float64 reference uses the exact erf, the kernel the A&S approximation (absolute
error < 1.5e-7), so the GEGLU bound adds |a| * (1.2 * 2^-20 * B_g + 1e-7 * |g|) + 2^-20 * B_a * |gelu(g)|.
An int8 output must equal clamp(rint(y64 * inv_scale)) except within that bound of a rounding tie, where it may be one
off."""
import os
import sys

import numpy as np
import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import w8a8_oracle as WQ  # noqa: E402

pytestmark = pytest.mark.gpu


def _f16_ulp(v):
    a = np.abs(v)
    e = np.floor(np.log2(np.maximum(a, 2.0 ** -14)))
    return 2.0 ** (e - 10)


def _linear_ref(x8, w8, cs, bias, residual, geglu, rows):
    """float64 (value, tolerance) [len(rows), N_out] of output rows `rows` of one int8 linear launch, before any int8
    rounding."""
    a = x8[rows].double()
    wd = w8.double()
    acc = a @ wd.t()
    y = acc.float().double() * cs.double()[None, :]
    mag = (a.abs() @ wd.abs().t()) * cs.double()[None, :]
    if bias is not None:
        y, mag = y + bias.double()[None, :], mag + bias.double().abs()[None, :]
    tol = 2.0 ** -20 * mag
    if geglu:
        av, gv, ma, mg = y[:, 0::2], y[:, 1::2], mag[:, 0::2], mag[:, 1::2]
        gel = gv * 0.5 * (1 + torch.erf(gv / np.sqrt(2.0)))
        y = av * gel
        tol = av.abs() * (1.2 * 2.0 ** -20 * mg + 1e-7 * gv.abs()) + 2.0 ** -20 * ma * gel.abs() + 2.0 ** -23 * y.abs()
    if residual is not None:
        r = residual[rows].double()
        y, tol = y + r, tol + 2.0 ** -23 * (y.abs() + r.abs())
    return y, tol


def _rows(m, max_rows):
    if m <= max_rows + 128:
        return torch.arange(m)
    pick = torch.randperm(m - 128, generator=torch.Generator().manual_seed(0))[:max_rows]
    return torch.cat([pick.sort().values, torch.arange(m - 128, m)])


def _check_q(q, y64, tol, inv, what):
    t = y64 * inv
    q64 = torch.clamp(torch.round(t), -127, 127)
    d = (q.double() - q64).abs()
    assert d.max() <= 1, f"{what}: |q - q64| = {d.max()}"
    near = ((t - torch.floor(t) - 0.5).abs() <= tol * inv + 1e-6) & (t.abs() < 127.5)
    assert not (d[~near] > 0).any(), f"{what}: {int((d[~near] > 0).sum())} values differ away from a rounding tie"


def _check_linear(x8, w8, cs, bias, residual, geglu, out, inv, what, max_rows=2048):
    m = out.shape[0]
    rows = _rows(m, max_rows)
    ref, tol = _linear_ref(x8.cpu(), w8.cpu(), cs.cpu(), None if bias is None else bias.cpu(),
                           None if residual is None else residual.cpu(), geglu, rows)
    got = out[rows.to(out.device)].cpu()
    if inv is not None:
        _check_q(got, ref, tol, inv, what)
        return
    ref, tol, got = ref.numpy(), tol.numpy(), got.double().numpy()
    bad = np.abs(got - ref) > _f16_ulp(ref) + tol
    idx = np.argwhere(bad)[:6]
    detail = ", ".join(f"[{int(rows[i])},{j}] ref={ref[i, j]!r} got={got[i, j]!r}" for i, j in idx)
    assert not bad.any(), f"{what}: {bad.sum()} of {bad.size} outputs off by more than the bound: {detail}"


# (m, c, n, geglu, bias, residual, int8 output, row statistics)
CASES = [
    (8192, 320, 960, False, False, False, False, False),     # attn1.to_q|k|v, SD-2.1 level 0
    (8192, 320, 320, False, True, False, False, True),       # proj_in before an fp16 qkv
    (2048, 640, 5120, True, True, False, True, False),       # GEGLU -> int8 ff.net.2
    (2048, 640, 5120, True, True, False, False, False),      # GEGLU -> fp16
    (512, 5120, 1280, False, True, True, True, False),       # last ff.net.2 -> int8 proj_out
    (512, 5120, 1280, False, True, True, False, True),       # ff.net.2 before an fp16 qkv
    (128, 1280, 1280, False, True, True, False, False),      # proj_out at 8x8 (split-K)
    (600, 48, 96, False, True, True, False, False),          # ragged rows, one k-block
]


@pytest.mark.parametrize("case", CASES)
def test_linear_s8_planned_launch_is_exact(cuda_lib, case):
    from b200sd import lib as L

    m, c, n, geglu, has_b, has_r, s8, rs = case
    dev = torch.device("cuda:0")
    g = torch.Generator().manual_seed(CASES.index(case))
    x8 = torch.randint(-127, 128, (m, c), generator=g, dtype=torch.int8).to(dev)
    w8 = torch.randint(-127, 128, (n, c), generator=g, dtype=torch.int8).to(dev)
    cs = (torch.rand(n, generator=g) * 1e-4 + 1e-6).to(dev)
    bias = torch.randn(n, generator=g).to(dev) if has_b else None
    n_out = n // 2 if geglu else n
    residual = torch.randn(m, n_out, generator=g).half().to(dev) if has_r else None
    inv = 127.0 / 4.0 if s8 else None
    st = {} if rs else None
    out = L.linear_s8(x8, w8, cs, bias, residual, geglu=geglu, out_inv_scale=inv, rowstats=st)
    out2 = L.linear_s8(x8, w8, cs, bias, residual, geglu=geglu, out_inv_scale=inv, rowstats={} if rs else None)
    torch.cuda.synchronize()
    assert out.dtype == (torch.int8 if s8 else torch.float16)
    assert torch.equal(out, out2)
    _check_linear(x8, w8, cs, bias, residual, geglu, out, inv, str(case))
    if rs:  # the row statistics are sums of the rounded fp16 outputs
        sums = st["rows"].sum(0).cpu().double()
        o = out.cpu().double()
        assert torch.allclose(sums[:, 0], o.sum(1), rtol=1e-5, atol=1e-2)
        assert torch.allclose(sums[:, 1], (o * o).sum(1), rtol=1e-5, atol=1e-2)


@pytest.mark.parametrize("shape", [(4096, 320), (2048, 640), (512, 1280), (77, 64)])
def test_layer_norm_s8_matches_fp64(cuda_lib, shape):
    from b200sd import lib as L

    rows, c = shape
    g = torch.Generator().manual_seed(rows + c)
    x = (torch.randn(rows, c, generator=g) * 2 + 0.3).half()
    gamma = torch.rand(c, generator=g) + 0.5
    beta = torch.randn(c, generator=g) * 0.2
    xd = x.double()
    mu = xd.mean(1, keepdim=True)
    y64 = (xd - mu) / torch.sqrt(((xd - mu) ** 2).mean(1, keepdim=True) + 1e-5) * gamma.double() + beta.double()
    inv = 127.0 / float(y64.abs().max()) * 1.3  # some values saturate
    q = L.layer_norm_s8(x.cuda(), gamma.cuda(), beta.cuda(), inv)
    torch.cuda.synchronize()
    _check_q(q.cpu(), y64, 1e-3 / inv, inv, str(shape))


@pytest.mark.parametrize("geglu", [False, True])
def test_fp16_linear_int8_output_matches_fp64(cuda_lib, geglu):
    """The fp16 GEMM's int8-output epilogue: ff.net.0.proj (GEGLU) or ff.net.2 (residual) in fp16 feeding a W8A8
    consumer.  Reference: the fp64 product of the fp16 operands, same epilogue."""
    from b200sd import lib as L

    g = torch.Generator().manual_seed(7 + geglu)
    m, c, n = 2048, 640, 5120 if geglu else 640
    x = (torch.randn(m, c, generator=g)).half()
    w = (torch.randn(n, c, generator=g) * c ** -0.5).half()
    bias = torch.randn(n, generator=g) * 0.1
    res = None if geglu else torch.randn(m, n, generator=g).half()
    inv = 127.0 / 6.0
    q = L.linear(x.cuda(), w.cuda(), bias.cuda(), None if res is None else res.cuda(), geglu=geglu, static_w=True,
                 out_inv_scale=inv)
    torch.cuda.synchronize()
    assert q.dtype == torch.int8
    y = x.double() @ w.double().t() + bias.double()
    mag = x.double().abs() @ w.double().abs().t() + bias.double().abs()
    tol = 2.0 ** -16 * mag  # fp32 accumulation of fp16 products in the tensor core's order
    if geglu:
        a, gv = y[:, 0::2], y[:, 1::2]
        gel = gv * 0.5 * (1 + torch.erf(gv / np.sqrt(2.0)))
        tol = a.abs() * (1.2 * tol[:, 1::2] + 1e-7 * gv.abs()) + tol[:, 0::2] * gel.abs()
        y = a * gel
    else:
        y = y + res.double()
    _check_q(q.cpu(), y, tol, inv, f"geglu={geglu}")


# ---------------------------------------------------------------------------------------------------------------------
# UNet
# ---------------------------------------------------------------------------------------------------------------------
def _unet_inputs(cfg, batch, hw, seed=2):
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(batch, 4, hw, hw, generator=g)
    ctx = torch.randn(batch, cfg["cross_attention_dim"], 1, 77, generator=g)
    t = torch.full((batch,), 501.0)
    return x, t, ctx


@pytest.mark.parametrize("model", ["tiny", "sd21"])
def test_unet_convs_and_linears_recipe_tracks_the_fake_quant_oracle(cuda_lib, model):
    """rms(engine - oracle_q) <= 1.5 * rms(oracle_q - oracle_fp32), the bound of test_w8a8_gpu.py's conv-only test,
    with every eligible convolution and transformer linear quantized (scales from an oracle calibration pass)."""
    from b200sd import config as C
    from b200sd import quantization as Q
    from b200sd.model import UNetModel
    from oracle import restated as R

    cfg, hw = (C.TINY_UNET, 16) if model == "tiny" else (C.SD21_BASE_UNET, 32)
    sd = {k: v.half().float() for k, v in C.random_state_dict(C.unet_param_shapes(cfg), seed=3).items()}
    x, t, ctx = _unet_inputs(cfg, 2, hw)
    x, ctx = x.half().float(), ctx.half().float()
    conv, lin = Q.quantizable_layers(cfg), Q.quantizable_linear_layers(cfg)
    with torch.no_grad():
        amax = WQ.calibrate(sd, cfg, x, t, ctx, set(conv) | set(lin))
    recipe = Q.W8A8Recipe.from_amax({k: amax[k] for k in conv}, cfg, {k: amax[k] for k in lin})
    with torch.no_grad():
        ref32 = R.unet_forward(sd, cfg, x, t, ctx)
        refq = WQ.unet_forward_q(sd, cfg, x, t, ctx, {**recipe.scales, **recipe.linear_scales})
    u = UNetModel(cfg, {k: v.half() for k, v in sd.items()}, batch=2, height=hw, width=hw, quantization=recipe)
    got = torch.from_numpy(u(sample=x.half().numpy(), timestep=t.half().numpy(),
                             encoder_hidden_states=ctx.half().numpy())["noise_pred"]).double()
    rms = lambda d: float(d.double().pow(2).mean().sqrt())  # noqa: E731
    e_engine, e_quant = rms(got - refq), rms(refq - ref32)
    print(f"{model}: engine-vs-q {e_engine:.4g}, q-vs-fp32 {e_quant:.4g}, ratio {e_engine / e_quant:.3f}")
    assert e_quant > 0 and e_engine <= 1.5 * e_quant, f"{model}: engine-vs-q {e_engine:.4g}, q-vs-fp32 {e_quant:.4g}"


def test_unet_partial_linear_recipe_mixes_int8_and_fp16_neighbours(cuda_lib):
    """Alternating int8 / fp16 launches inside the transformers (fp16 LayerNorm folds after int8 producers, fp16 GEGLU
    and ff.net.2 writing int8 operands) track the fake-quant oracle like the full recipe."""
    from b200sd import config as C
    from b200sd import quantization as Q
    from b200sd.model import UNetModel
    from oracle import restated as R

    cfg, hw = C.TINY_UNET, 16
    sd = {k: v.half().float() for k, v in C.random_state_dict(C.unet_param_shapes(cfg), seed=4).items()}
    x, t, ctx = _unet_inputs(cfg, 2, hw, seed=5)
    x, ctx = x.half().float(), ctx.half().float()
    lin = Q.quantizable_linear_layers(cfg)
    # down blocks: int8 proj_in / attn2.to_q / ff.net.2 beside fp16 qkv and GEGLU; up blocks: int8 qkv and GEGLU beside
    # fp16 proj_in and ff.net.2; mid block: fp16 ff.net.2 writing the int8 operand of proj_out
    pick = [n for n in lin if (n.startswith("down_blocks") and n.endswith((".proj_in", ".attn2.to_q", ".ff.net.2")))
            or (n.startswith("up_blocks") and n.endswith((".to_q", ".to_k", ".to_v", ".ff.net.0.proj"))
                and ".attn2." not in n)
            or n == "mid_block.attentions.0.proj_out"]
    with torch.no_grad():
        amax = WQ.calibrate(sd, cfg, x, t, ctx, set(pick))
        ref32 = R.unet_forward(sd, cfg, x, t, ctx)
        recipe = Q.W8A8Recipe({}, Q.architecture(cfg), {k: amax[k] / 127 for k in pick})
        refq = WQ.unet_forward_q(sd, cfg, x, t, ctx, recipe.linear_scales)
    recipe.validate(cfg)
    u = UNetModel(cfg, {k: v.half() for k, v in sd.items()}, batch=2, height=hw, width=hw, quantization=recipe)
    got = torch.from_numpy(u(sample=x.half().numpy(), timestep=t.half().numpy(),
                             encoder_hidden_states=ctx.half().numpy())["noise_pred"])
    rms = lambda d: float(d.double().pow(2).mean().sqrt())  # noqa: E731
    e_engine, e_quant = rms(got.double() - refq.double()), rms(refq.double() - ref32.double())
    print(f"tiny partial: engine-vs-q {e_engine:.4g}, q-vs-fp32 {e_quant:.4g}")
    assert e_quant > 0 and e_engine <= 1.5 * e_quant, f"engine-vs-q {e_engine:.4g}, q-vs-fp32 {e_quant:.4g}"


_FUSION_ENV = ("B200SD_FUSED", "B200SD_HALO_TMA", "B200SD_FOLD_SC", "B200SD_CLUSTER_SPLITK", "B200SD_SMEM_KB",
               "B200SD_STAGED", "B200SD_TILED_W")


@pytest.mark.parametrize("name", ["sd21_b2", "sd15_b2", "sdxl_1024_b2"])
def test_every_int8_linear_launch_of_the_w8a8_models_is_exact(cuda_lib, monkeypatch, name):
    """Convs + linears W8A8 SD-2.1-base and SD-1.5 at 512^2 and SDXL at 1024^2 (random init, batch 2), scales from a
    calibration pass of the fp16 engine on the same inputs.  Every linear_s8 launch of one forward is recorded and
    replayed on the CPU (a sample of 512 rows plus the tail tile per launch)."""
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
    slots = m.engine.set_calibration(True, linear=True)
    m(**inputs)
    lin = Q.quantizable_linear_layers(cfg)
    amax = {k: float(v) for k, v in slots.items()}
    recipe = Q.W8A8Recipe.from_amax({k: v for k, v in amax.items() if k not in lin}, cfg,
                                    {k: v for k, v in amax.items() if k in lin})
    assert len(recipe.linear_scales) == len(lin)
    del m, slots
    torch.cuda.empty_cache()
    sd = C.random_state_dict(C.unet_param_shapes(cfg), seed=5, dtype=torch.float16)
    qm = UNetModel(cfg, sd, batch=batch, height=lat_h, width=lat_w, use_cuda_graph=False, quantization=recipe)
    del sd
    calls = []
    orig = L.linear_s8

    def record(x, wgt, col_scale, bias=None, residual=None, **kw):
        o = orig(x, wgt, col_scale, bias, residual, **kw)
        calls.append((x, wgt, col_scale, bias, residual, kw.get("geglu", False), kw.get("out_inv_scale"), o))
        return o

    monkeypatch.setattr(L, "linear_s8", record)
    out = qm(**inputs)["noise_pred"]
    torch.cuda.synchronize()
    assert np.isfinite(out).all()
    n_tr = sum(1 for n in lin if n.endswith(".proj_in"))
    n_blk = sum(1 for n in lin if n.endswith(".ff.net.2"))
    assert len(calls) == 2 * n_tr + 4 * n_blk, (len(calls), n_tr, n_blk)
    for i, (x8, w8, cs, bias, residual, geglu, inv, o) in enumerate(calls):
        _check_linear(x8, w8, cs, bias, residual, geglu, o, inv, f"{name} launch {i} {tuple(x8.shape)}x{tuple(w8.shape)}",
                      max_rows=512)


def test_pipeline_linear_calibration_saved_recipe_and_loop_graph(cuda_lib, tmp_path):
    """calibrate_unet(linear=True) -> saved v2 recipe -> from_pretrained(unet_quantization=path) generates images; the
    loop graph is bit-identical to the step-by-step path."""
    import test_factory_gpu as TF
    from b200sd import config as C
    from b200sd import quantization as Q
    from b200sd.pipeline import B200StableDiffusionPipeline as P

    TF._model_dir(tmp_path, C.TINY_UNET, seed=11)
    pipe = P.from_pretrained(str(tmp_path), height=64, width=64)
    recipe = pipe.calibrate_unet(["a red cube"], num_inference_steps=3, seed=2, linear=True)
    assert len(recipe.scales) == len(Q.quantizable_layers(C.TINY_UNET))
    assert len(recipe.linear_scales) == len(Q.quantizable_linear_layers(C.TINY_UNET))
    assert all(s > 0 for s in recipe.linear_scales.values())
    path = tmp_path / "w8a8.json"
    recipe.save(path)
    qpipe = P.from_pretrained(str(tmp_path), height=64, width=64, unet_quantization=str(path))
    kw = dict(height=64, width=64, num_inference_steps=3, guidance_scale=5.0, output_type="np", seed=7)
    img = qpipe("a red cube", **kw).images
    ref = pipe("a red cube", **kw).images
    assert img.shape == ref.shape == (1, 64, 64, 3) and np.isfinite(img).all()
    assert not np.array_equal(img, ref)
    u = qpipe.unet
    lat = torch.from_numpy(np.random.RandomState(0).randn(1, 4, u.h, u.w).astype(np.float32))
    emb = torch.from_numpy(np.random.RandomState(1).randn(2, C.TINY_UNET["cross_attention_dim"], 1, 77).astype(np.float16))
    a = qpipe.denoise(emb, lat, 4, 7.5).clone()
    b = qpipe.denoise(emb, lat, 4, 7.5, record=[]).clone()  # step by step
    assert torch.isfinite(a).all() and torch.equal(a, b), "loop graph and step-by-step path differ"
