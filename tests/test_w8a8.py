"""CPU tests of the W8A8 convolution path: the int8 kernels' machine code, the int8 planner on every quantizable launch
of the shipped models, the quantization arithmetic and recipes, and a float64 fake-quant oracle."""
import json
import math
import os
import re
import shutil
import subprocess
import sys

import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import w8a8_oracle as WQ  # noqa: E402

WIDTHS = (256, 192, 160, 128, 96, 64, 32, 16)
SMEM_LIMIT = 227 * 1024


def _sass_functions(path):
    cuobjdump = shutil.which("cuobjdump") or "/usr/local/cuda/bin/cuobjdump"
    if not os.path.exists(cuobjdump):
        pytest.skip("cuobjdump not available")
    sass = subprocess.run([cuobjdump, "-sass", path], capture_output=True, text=True, check=True).stdout
    for chunk in re.split(r"\n\s*Function : ", sass)[1:]:
        name, body = chunk.split("\n", 1)
        yield name.strip(), body


def test_int8_conv_kernels_use_igmma_pipelined_without_spills():
    import __graft_entry__ as ge
    from b200sd import lib

    ge.build()
    kernels = {n: b for n, b in _sass_functions(lib.lib_path()) if "igmma_conv_kernel" in n}
    # generic variant at all eight widths, plain and split-K at the seven widths >= 32
    assert len(kernels) == 8 + 7 + 7, sorted(kernels)
    for name, body in kernels.items():
        assert "wgmma_gemm_kernel" not in name
        igmma = re.findall(r"\bIGMMA\.64x(\d+)x32\.S8\.S8", body)
        assert igmma, name
        wait0 = len(re.findall(r"WARPGROUP\.DEPBAR\.LE gsb0, 0x0\b", body))
        wait_n = len(re.findall(r"WARPGROUP\.DEPBAR\.LE gsb0, 0x[1-9a-f]", body))
        assert wait_n >= 1 and wait0 <= 2, f"{name}: {len(igmma)} IGMMA, {wait0} waits for 0, {wait_n} waits for > 0"
        assert not re.findall(r"\b(LDL|STL)(\.\w+)*\b", body), f"{name}: local-memory (spill) instructions"
        assert not re.findall(r"\bHGMMA\.", body), name


# ---------------------------------------------------------------------------------------------------------------------
# planner
# ---------------------------------------------------------------------------------------------------------------------
def _plan_fields(s):
    return {k: int(v) if re.fullmatch(r"-?\d+", v) else v for k, v in (kv.split("=") for kv in s.split())}


def _shipped_int8_launches():
    """(model, layer, Cin, Cout, hw) of every int8 convolution launch: each ResNet conv1 / conv2 and up-sampler
    convolution of SD-2.1-base and SD-1.5 at 512^2, SD-2.1 at 768^2 and SDXL at 768^2 / 1024^2, batch 2."""
    from b200sd import config as C
    from b200sd import quantization as Q

    models = {"sd21_512": (C.SD21_BASE_UNET, 64), "sd15_512": (C.SD15_UNET, 64), "sd21_768": (C.SD21_UNET, 96),
              "sdxl_768": (C.SDXL_BASE_UNET, 96), "sdxl_1024": (C.SDXL_BASE_UNET, 128)}
    out = []
    for m, (cfg, hw0) in models.items():
        boc = list(cfg["block_out_channels"])
        nb = len(boc)
        for name, cin in Q.quantizable_layers(cfg).items():
            part = name.split(".")
            if part[0] == "mid_block":
                lvl, cout = nb - 1, boc[-1]
            elif part[0] == "down_blocks":
                lvl, cout = int(part[1]), boc[int(part[1])]
            else:  # up block i runs at level nb - 1 - i; its up-sampler convolution one level up
                i = int(part[1])
                lvl, cout = nb - 1 - i - (1 if "upsamplers" in name else 0), boc[::-1][i]
            out.append((m, name, cin, cout, hw0 >> lvl))
    return out


LAUNCHES = _shipped_int8_launches()


def test_int8_launch_list_covers_the_models():
    names = {(m, n) for m, n, *_ in LAUNCHES}
    assert ("sd21_512", "up_blocks.3.resnets.0.conv1") in names and ("sdxl_1024", "up_blocks.1.upsamplers.0.conv") in names
    by = {(m, n): (cin, cout, hw) for m, n, cin, cout, hw in LAUNCHES}
    assert by[("sd21_512", "up_blocks.3.resnets.0.conv1")] == (960, 320, 64)
    assert by[("sd21_512", "up_blocks.3.resnets.1.conv1")] == (640, 320, 64)
    assert by[("sd21_512", "up_blocks.0.upsamplers.0.conv")] == (1280, 1280, 16)
    assert by[("sdxl_1024", "up_blocks.2.resnets.0.conv1")] == (960, 320, 128)
    assert by[("sd21_512", "mid_block.resnets.1.conv2")] == (1280, 1280, 8)


@pytest.mark.parametrize("model", sorted({m for m, *_ in LAUNCHES}))
def test_int8_planner_gives_a_valid_plan_for_every_launch(model):
    from b200sd import lib

    lib.load()
    for m, name, cin, cout, hw in LAUNCHES:
        if m != model:
            continue
        conv1 = name.endswith("conv1")
        p = _plan_fields(lib.describe_plan_s8(cout, cin, 2, hw, hw, bias_rows=hw * hw if conv1 else 0,
                                              has_residual=name.endswith("conv2")))
        bn, sp, kb, kps, st = p["block_n"], p["splits"], p["kb_total"], p["kb_per_split"], p["stages"]
        assert bn in WIDTHS, (name, p)
        assert kb == 9 * math.ceil(cin / 128), (name, p)
        per_stage = 128 * 128 + bn * 128
        assert 2 <= st <= 8 and st * per_stage + p["epi_smem"] + 1024 <= SMEM_LIMIT, (name, p)
        assert st * per_stage >= 128 * (bn + 4) * 4, (name, p)  # the fp32 tile parks over the stages
        if p["cluster"]:
            assert sp in (2, 4, 8) and sp <= kb, (name, p)
        else:
            assert sp * kps >= kb and (sp - 1) * kps < kb, (name, p)
        assert p["variant"] in (0, 1, 4) and p["staged"] == 0, (name, p)
        assert p["n_tiles"] * bn >= cout


@pytest.mark.parametrize("field,kw", [
    ("mode", dict(mode=0)), ("stride", dict(stride=2)), ("a1", dict(c1=64)), ("geglu", dict(geglu=1)),
    ("act", dict(act=1)), ("out_f32", dict(out_f32=1)), ("halo", dict(halo=1)), ("upsample2x", dict(upsample2x=1)),
    ("gn_", dict(gn_groups=32)), ("cs_", dict(cs_partial=1)), ("rs_out", dict(rs_out=1)), ("ln_", dict(ln_parts=1)),
    ("a2 / a3", dict(c2=64)), ("pad_after_only", dict(pad_after_only=1)),
])
def test_int8_planner_rejects_unsupported_fields_by_name(field, kw):
    from b200sd import lib

    lib.load()
    a = lib.GemmArgs()
    a.mode, a.n, a.c0, a.n_img, a.h, a.w, a.stride = 1, 320, 320, 2, 16, 16, 1
    for k, v in kw.items():
        setattr(a, k, v)
    with pytest.raises(lib.B200SDError, match=re.escape(field)):
        lib.plan_ex_s8(a)


def test_int8_weight_tiling_layout():
    from b200sd import lib

    g = torch.Generator().manual_seed(0)
    cin, cout, bn = 320, 96, 32
    w = torch.randint(-127, 128, (cout, 9 * cin), generator=g, dtype=torch.int8)
    t = lib.pack_tiled(w, cin, 0, 9, bn, chunk=128)
    kc = math.ceil(cin / 128)
    assert t.shape == (cout // bn, 9 * kc, bn, 128) and t.dtype == torch.int8
    w3 = w.reshape(cout, 9, cin)
    for nt in range(cout // bn):
        for tap in range(9):
            for j in range(kc):
                lo, hi = 128 * j, min(128 * j + 128, cin)
                blk = t[nt, tap * kc + j]
                assert torch.equal(blk[:, : hi - lo], w3[nt * bn:(nt + 1) * bn, tap, lo:hi])
                assert not blk[:, hi - lo:].any()


# ---------------------------------------------------------------------------------------------------------------------
# quantization arithmetic and recipes
# ---------------------------------------------------------------------------------------------------------------------
def test_weight_scales_rounding_and_saturation():
    from b200sd import quantization as Q

    w = torch.tensor([[1.0, -2.0, 0.5, 127.0 / 127 * 2], [0.0, 0.0, 0.0, 0.0], [2.5, -2.5, 1.5, 127.0]])
    q, s = Q.quantize_weight(w)
    assert torch.allclose(s, torch.tensor([2.0 / 127, 1.0, 1.0]))
    assert q.dtype == torch.int8
    assert q[0].tolist() == [64, -127, 32, 127]  # 63.5 -> 64 (half to even), 31.75 -> 32
    assert q[1].tolist() == [0, 0, 0, 0]
    assert q[2].tolist() == [2, -2, 2, 127]  # 2.5 -> 2, -2.5 -> -2, 1.5 -> 2: round half to even
    x = torch.tensor([0.5, 1.5, -0.5, 300.0, -300.0, 126.6])
    assert Q.quantize_activation(x, 1.0).tolist() == [0, 2, -0, 127, -127, 127]


def _tiny_cfg():
    from b200sd import config as C
    return C.TINY_UNET


def test_quantizable_layers_of_sd21():
    from b200sd import config as C
    from b200sd import quantization as Q

    layers = Q.quantizable_layers(C.SD21_BASE_UNET)
    assert len(layers) == 2 * (4 * 2 + 2 + 4 * 3) + 3
    assert layers["up_blocks.0.resnets.0.conv1"] == 2560 and layers["up_blocks.3.resnets.2.conv1"] == 640
    assert layers["down_blocks.1.resnets.0.conv1"] == 320 and layers["down_blocks.1.resnets.0.conv2"] == 640


def test_recipe_json_round_trip_and_validation(tmp_path):
    from b200sd import quantization as Q

    cfg = _tiny_cfg()
    layers = Q.quantizable_layers(cfg)
    r = Q.W8A8Recipe.from_amax({n: 1.0 + i for i, n in enumerate(layers)}, cfg)
    p = tmp_path / "r.json"
    r.save(p)
    r2 = Q.W8A8Recipe.load(p)
    assert r2.scales == r.scales and r2.arch == r.arch
    assert r2.validate(cfg) == layers
    assert Q.as_recipe(str(p)).scales == r.scales


@pytest.mark.parametrize("bad,match", [
    ({"mid_block.attentions.0.proj_in": 0.1}, "mid_block.attentions.0.proj_in"),
    ({"down_blocks.0.downsamplers.0.conv": 0.1}, "down_blocks.0.downsamplers.0.conv"),
    ({"conv_in": 0.1}, "conv_in"),
    ({"up_blocks.7.resnets.0.conv1": 0.1}, "up_blocks.7.resnets.0.conv1"),
    ({"up_blocks.0.resnets.0.conv1": 0.0}, "up_blocks.0.resnets.0.conv1"),
    ({"up_blocks.0.resnets.0.conv2": float("nan")}, "up_blocks.0.resnets.0.conv2"),
    ({"mid_block.resnets.0.conv1": float("inf")}, "mid_block.resnets.0.conv1"),
])
def test_recipe_rejects_bad_layers(bad, match):
    from b200sd import quantization as Q

    with pytest.raises(ValueError, match=re.escape(match)):
        Q.W8A8Recipe(bad, Q.architecture(_tiny_cfg())).validate(_tiny_cfg())


def test_recipe_rejects_another_architecture():
    from b200sd import config as C
    from b200sd import quantization as Q

    r = Q.W8A8Recipe({"mid_block.resnets.0.conv1": 0.1}, Q.architecture(C.SD21_BASE_UNET))
    with pytest.raises(ValueError, match="block_out_channels"):
        r.validate(_tiny_cfg())


def test_reference_sensitivity_json_selects_by_conv_psnr(tmp_path):
    from b200sd import quantization as Q

    cfg = _tiny_cfg()
    layers = list(Q.quantizable_layers(cfg))
    cal = Q.W8A8Recipe.from_amax({n: 2.0 for n in layers}, cfg)
    sens = {"conv": {layers[0]: 41.0, layers[1]: 30.0, layers[2]: 35.0, "conv_in": 50.0,
                     "down_blocks.0.attentions.0.proj_in": 60.0},
            "einsum": {"down_blocks.0.attentions.0.transformer_blocks.0.attn1.einsum": 50.0},
            "model_version": "stabilityai/stable-diffusion-2-1-base"}
    p = tmp_path / "s.json"
    p.write_text(json.dumps(sens))
    recipe, kept = Q.select_from_sensitivity(str(p), 35.0, cal)
    assert sorted(recipe.scales) == sorted([layers[0], layers[2]])
    assert recipe.scales[layers[0]] == pytest.approx(2.0 / 127)
    assert kept == sorted([layers[1], "conv_in", "down_blocks.0.attentions.0.proj_in",
                           "down_blocks.0.attentions.0.transformer_blocks.0.attn1.einsum"])


# ---------------------------------------------------------------------------------------------------------------------
# fake-quant oracle
# ---------------------------------------------------------------------------------------------------------------------
def _tiny_inputs(cfg, seed=3):
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(2, 4, 8, 8, generator=g, dtype=torch.float64)
    ctx = torch.randn(2, cfg["cross_attention_dim"], 1, 7, generator=g, dtype=torch.float64)
    t = torch.tensor([981.0, 981.0])
    return x, t, ctx


def test_fake_quant_oracle_with_empty_recipe_is_the_oracle():
    from b200sd import config as C
    from oracle import restated as R

    cfg = _tiny_cfg()
    sd = C.random_state_dict(C.unet_param_shapes(cfg), seed=1)
    x, t, ctx = _tiny_inputs(cfg)
    ref = R.unet_forward(sd, cfg, x.float(), t, ctx.float())
    got = WQ.unet_forward_q(sd, cfg, x.float(), t, ctx.float(), {})
    assert torch.equal(ref, got)


def test_fake_quant_conv_is_the_exact_integer_product_times_scales():
    g = torch.Generator().manual_seed(4)
    w = torch.randn(24, 32, 3, 3, generator=g, dtype=torch.float64)
    b = torch.randn(24, generator=g, dtype=torch.float64)
    x = torch.randn(2, 32, 6, 5, generator=g, dtype=torch.float64)
    s_a = float(x.abs().max()) / 127 * 0.8  # some saturation
    out = WQ.qconv(x, w, b, s_a)
    qa = torch.clamp(torch.round(x / s_a), -127, 127).to(torch.int64)
    s_w = w.reshape(24, -1).abs().amax(1) / 127
    qw = torch.clamp(torch.round(w / s_w[:, None, None, None]), -127, 127).to(torch.int64)
    xp = torch.nn.functional.pad(qa, (1, 1, 1, 1))
    acc = torch.zeros(2, 24, 6, 5, dtype=torch.int64)
    for dy in range(3):
        for dx in range(3):
            acc += torch.einsum("nchw,oc->nohw", xp[:, :, dy:dy + 6, dx:dx + 5], qw[:, :, dy, dx])
    ref = acc.double() * (s_a * s_w)[None, :, None, None] + b[None, :, None, None]
    assert torch.equal(out, ref)


@pytest.mark.parametrize("var,value", [("B200SD_FUSED", "1"), ("B200SD_FUSED", "0"), ("B200SD_HALO_TMA", "1024")])
def test_recipe_rejects_the_opt_in_paths_by_variable(monkeypatch, var, value):
    """Checked before anything is allocated on a device."""
    from b200sd import config as C
    from b200sd import quantization as Q
    from b200sd.unet import UNetEngine

    cfg = _tiny_cfg()
    recipe = Q.W8A8Recipe({"mid_block.resnets.0.conv1": 0.1}, Q.architecture(cfg))
    monkeypatch.setenv(var, value)
    with pytest.raises(ValueError, match=var):
        UNetEngine(cfg, {}, device="cpu", quantization=recipe)
