"""CPU tests of the W8A8 transformer linears: the int8 linear and int8-output kernels' machine code, the planner on every
linear launch of the shipped models, the layer list, the recipe's linear section and the sensitivity-JSON selection."""
import json
import math
import os
import re
import shutil
import subprocess

import pytest

WIDTHS = (256, 192, 160, 128, 96, 64, 32)
SMEM_LIMIT = 227 * 1024


def _sass_functions(path):
    cuobjdump = shutil.which("cuobjdump") or "/usr/local/cuda/bin/cuobjdump"
    if not os.path.exists(cuobjdump):
        pytest.skip("cuobjdump not available")
    sass = subprocess.run([cuobjdump, "-sass", path], capture_output=True, text=True, check=True).stdout
    for chunk in re.split(r"\n\s*Function : ", sass)[1:]:
        name, body = chunk.split("\n", 1)
        yield name.strip(), body


def test_int8_linear_and_int8_output_kernels_are_pipelined_without_spills():
    import __graft_entry__ as ge
    from b200sd import lib

    ge.build()
    funcs = dict(_sass_functions(lib.lib_path()))
    lin = {n: b for n, b in funcs.items() if "igmma_linear_kernel" in n}
    s8out = {n: b for n, b in funcs.items() if "wgmma_gemm_s8out_kernel" in n}
    # (GEGLU, fp16 out), (plain, int8 out), (GEGLU, int8 out) / (plain, GEGLU) with int8 output, at the widths >= 32
    assert len(lin) == 3 * 7 and len(s8out) == 2 * 7, (sorted(lin), sorted(s8out))
    for name, body in {**lin, **s8out}.items():
        mma = re.findall(r"\bIGMMA\.64x(\d+)x32\.S8\.S8" if name in lin else r"\bHGMMA\.64x(\d+)x16\.F32\b(?!\.BF16)", body)
        assert mma, name
        assert not re.findall(r"\bHGMMA\." if name in lin else r"\bIGMMA\.", body), name
        wait0 = len(re.findall(r"WARPGROUP\.DEPBAR\.LE gsb0, 0x0\b", body))
        wait_n = len(re.findall(r"WARPGROUP\.DEPBAR\.LE gsb0, 0x[1-9a-f]", body))
        assert wait_n >= 1 and wait0 <= 2, f"{name}: {len(mma)} MMA, {wait0} waits for 0, {wait_n} waits for > 0"
        assert not re.findall(r"\b(LDL|STL)(\.\w+)*\b", body), f"{name}: local-memory (spill) instructions"
    ln = {n: b for n, b in funcs.items() if "layer_norm_s8_kernel" in n}
    assert len(ln) == 3, sorted(ln)
    for name, body in ln.items():
        assert not re.findall(r"\b(LDL|STL)(\.\w+)*\b", body), name


# ---------------------------------------------------------------------------------------------------------------------
# layer list
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("model,count,spot", [
    ("SD15_UNET", 16 * 8, {"down_blocks.0.attentions.0.proj_in": 320,
                           "mid_block.attentions.0.transformer_blocks.0.ff.net.2": 5120,
                           "up_blocks.3.attentions.2.proj_out": 320}),
    ("SD21_BASE_UNET", 16 * 8, {"down_blocks.2.attentions.1.transformer_blocks.0.attn1.to_v": 1280,
                                "up_blocks.1.attentions.0.transformer_blocks.0.ff.net.0.proj": 1280}),
    ("SD21_UNET", 16 * 8, {"up_blocks.2.attentions.1.transformer_blocks.0.attn2.to_q": 640}),
    # SDXL: 11 transformers with 2 + 2*10 + 10 + 3*10 + 3*2 = 70 blocks
    ("SDXL_BASE_UNET", 11 * 2 + 70 * 6, {"down_blocks.2.attentions.1.transformer_blocks.9.ff.net.2": 5120,
                                         "mid_block.attentions.0.transformer_blocks.9.attn1.to_q": 1280,
                                         "up_blocks.1.attentions.2.transformer_blocks.1.ff.net.0.proj": 640,
                                         "down_blocks.1.attentions.0.proj_in": 640}),
])
def test_quantizable_linear_layers(model, count, spot):
    from b200sd import config as C
    from b200sd import quantization as Q

    layers = Q.quantizable_linear_layers(getattr(C, model))
    assert len(layers) == count
    for name, cin in spot.items():
        assert layers[name] == cin, name
    assert not any(re.search(r"to_out|attn2\.to_[kv]|conv|time_emb", n) for n in layers)
    assert "down_blocks.0.attentions.0.proj_in" not in Q.quantizable_linear_layers(C.SDXL_BASE_UNET)  # no attention there
    assert "up_blocks.0.attentions.0.transformer_blocks.9.ff.net.2" in Q.quantizable_linear_layers(C.SDXL_BASE_UNET)


# ---------------------------------------------------------------------------------------------------------------------
# recipe
# ---------------------------------------------------------------------------------------------------------------------
def _tiny():
    from b200sd import config as C
    return C.TINY_UNET


def test_recipe_v1_bytes_unchanged_and_v2_round_trip(tmp_path):
    from b200sd import quantization as Q

    cfg = _tiny()
    conv = {n: 1.0 + i for i, n in enumerate(Q.quantizable_layers(cfg))}
    v1 = Q.W8A8Recipe.from_amax(conv, cfg)
    v1.save(tmp_path / "v1.json")
    want = json.dumps({"format": "b200sd-w8a8", "version": 1, "architecture": Q.architecture(cfg),
                       "activation_scales": {k: v / 127.0 for k, v in conv.items()}}, indent=1, sort_keys=True)
    assert (tmp_path / "v1.json").read_text() == want
    r1 = Q.W8A8Recipe.load(tmp_path / "v1.json")
    assert r1.scales == v1.scales and r1.linear_scales == {}

    lin = {n: 2.0 + i for i, n in enumerate(Q.quantizable_linear_layers(cfg))}
    for n in list(lin):  # one input: one scale per attn1 triple
        if n.endswith((".to_k", ".to_v")):
            lin[n] = lin[n.rsplit(".", 1)[0] + ".to_q"]
    v2 = Q.W8A8Recipe.from_amax(conv, cfg, lin)
    v2.save(tmp_path / "v2.json")
    d = json.loads((tmp_path / "v2.json").read_text())
    assert d["version"] == 2 and len(d["linear_activation_scales"]) == len(lin)
    r2 = Q.W8A8Recipe.load(tmp_path / "v2.json")
    assert r2.scales == v2.scales and r2.linear_scales == v2.linear_scales
    assert r2.validate(cfg) == Q.quantizable_layers(cfg)
    assert r2.validate_linear(cfg) == Q.quantizable_linear_layers(cfg)


def _blk(i=0):
    return f"down_blocks.0.attentions.0.transformer_blocks.{i}"


@pytest.mark.parametrize("lin,match", [
    ({_blk() + ".attn1.to_out.0": 0.1}, "to_out.0"),
    ({_blk() + ".attn2.to_out.0": 0.1}, "attn2.to_out.0"),
    ({_blk() + ".attn2.to_k": 0.1}, "attn2.to_k"),
    ({_blk() + ".attn2.to_v": 0.1}, "attn2.to_v"),
    ({"down_blocks.1.resnets.0.conv_shortcut": 0.1}, "conv_shortcut"),
    ({"down_blocks.0.resnets.0.time_emb_proj": 0.1}, "time_emb_proj"),
    ({"conv_in": 0.1}, "conv_in"),
    ({"down_blocks.0.downsamplers.0.conv": 0.1}, "down_blocks.0.downsamplers.0.conv"),
    ({_blk() + ".attn1.to_q": 0.1, _blk() + ".attn1.to_k": 0.1}, _blk() + ".attn1.to_v"),
    ({_blk() + ".attn1.to_q": 0.1, _blk() + ".attn1.to_k": 0.1, _blk() + ".attn1.to_v": 0.2}, "one activation scale"),
    ({_blk() + ".ff.net.2": 0.0}, _blk() + ".ff.net.2"),
    ({_blk() + ".ff.net.0.proj": float("nan")}, _blk() + ".ff.net.0.proj"),
    ({"mid_block.attentions.0.proj_out": float("inf")}, "mid_block.attentions.0.proj_out"),
    ({"mid_block.attentions.0.proj_in": -1.0}, "mid_block.attentions.0.proj_in"),
    ({"down_blocks.0.attentions.0.transformer_blocks.7.ff.net.2": 0.1}, "transformer_blocks.7.ff.net.2"),
])
def test_recipe_rejects_bad_linear_layers_by_name(lin, match):
    from b200sd import quantization as Q

    r = Q.W8A8Recipe({}, Q.architecture(_tiny()), lin)
    with pytest.raises(ValueError, match=re.escape(match)):
        r.validate(_tiny())


def test_sensitivity_selection_with_linear(tmp_path):
    """A README-shaped sensitivity JSON: every Conv2d of the reference UNet (its linears are 1x1 convolutions) -> PSNR."""
    from b200sd import quantization as Q

    cfg = _tiny()
    conv = list(Q.quantizable_layers(cfg))
    lin = Q.quantizable_linear_layers(cfg)
    cal = Q.W8A8Recipe.from_amax({n: 2.0 for n in conv}, cfg, {n: 4.0 for n in lin})
    b0, b1 = "down_blocks.0.attentions.0.transformer_blocks.0", "down_blocks.0.attentions.1.transformer_blocks.0"
    psnr = {conv[0]: 45.0, conv[1]: 30.0,
            "down_blocks.0.attentions.0.proj_in": 49.8, "down_blocks.0.attentions.0.proj_out": 37.9,
            b0 + ".attn1.to_q": 44.1, b0 + ".attn1.to_k": 41.3, b0 + ".attn1.to_v": 38.6,   # triple passes
            b1 + ".attn1.to_q": 43.0, b1 + ".attn1.to_k": 36.0, b1 + ".attn1.to_v": 40.0,   # one member fails
            b0 + ".attn1.to_out.0": 50.0, b0 + ".attn2.to_q": 39.0, b0 + ".attn2.to_k": 60.0,
            b0 + ".ff.net.0.proj": 42.0, b0 + ".ff.net.2": 37.0, "conv_in": 50.0}
    sens = {"conv": psnr, "einsum": {b0 + ".attn1.einsum": 50.0}, "model_version": "stabilityai/stable-diffusion-2-1-base"}
    p = tmp_path / "s.json"
    p.write_text(json.dumps(sens))

    r0, kept0 = Q.select_from_sensitivity(str(p), 38.0, cal)  # without linear=True: the convolutions only
    assert sorted(r0.scales) == [conv[0]] and r0.linear_scales == {}
    assert "down_blocks.0.attentions.0.proj_in" in kept0

    r, kept = Q.select_from_sensitivity(str(p), 38.0, cal, linear=True)
    assert sorted(r.scales) == [conv[0]]
    assert sorted(r.linear_scales) == sorted(["down_blocks.0.attentions.0.proj_in", b0 + ".attn1.to_q",
                                              b0 + ".attn1.to_k", b0 + ".attn1.to_v", b0 + ".attn2.to_q",
                                              b0 + ".ff.net.0.proj"])
    assert all(v == pytest.approx(4.0 / 127) for v in r.linear_scales.values())
    assert kept == sorted([conv[1], "down_blocks.0.attentions.0.proj_out", b1 + ".attn1.to_q", b1 + ".attn1.to_k",
                           b1 + ".attn1.to_v", b0 + ".attn1.to_out.0", b0 + ".attn2.to_k", b0 + ".ff.net.2", "conv_in",
                           b0 + ".attn1.einsum"])
    assert r.validate(cfg)  is not None  # a valid recipe


# ---------------------------------------------------------------------------------------------------------------------
# planner
# ---------------------------------------------------------------------------------------------------------------------
def _plan_fields(s):
    return {k: int(v) if re.fullmatch(r"-?\d+", v) else v for k, v in (kv.split("=") for kv in s.split())}


MODELS = {"sd21_512": ("SD21_BASE_UNET", 64), "sd15_512": ("SD15_UNET", 64), "sd21_768": ("SD21_UNET", 96),
          "sdxl_768": ("SDXL_BASE_UNET", 96), "sdxl_1024": ("SDXL_BASE_UNET", 128)}


def _linear_launches(model):
    """(what, kwargs) of every int8-linear / int8-output launch kind of one transformer level, batch 2: the launches of a
    convs + linears recipe and of the partial recipes (fp16 neighbours that read or write the int8 operands)."""
    from b200sd import config as C
    from b200sd import quantization as Q

    name, hw0 = MODELS[model]
    cfg = getattr(C, name)
    nb = len(cfg["block_out_channels"])
    seen = set()
    for p, c, _ in Q._transformers(cfg):
        part = p.split(".")
        lvl = int(part[1]) if part[0] == "down_blocks" else (nb - 1 if part[0] == "mid_block" else nb - 1 - int(part[1]))
        m = 2 * (hw0 >> lvl) ** 2
        if (m, c) in seen:
            continue
        seen.add((m, c))
        yield "s8", dict(m=m, n=c, c0=c)                                        # proj_in
        yield "s8", dict(m=m, n=c, c0=c, rowstats=True)                         # proj_in before an fp16 qkv
        yield "s8", dict(m=m, n=3 * c, c0=c, has_bias=False)                    # attn1.to_q|k|v
        yield "s8", dict(m=m, n=c, c0=c, has_bias=False)                        # attn2.to_q
        yield "s8", dict(m=m, n=8 * c, c0=c, geglu=True)                        # ff.net.0.proj -> fp16
        yield "s8", dict(m=m, n=8 * c, c0=c, geglu=True, out_s8=True)           # ff.net.0.proj -> int8
        yield "s8", dict(m=m, n=c, c0=4 * c, has_residual=True)                 # ff.net.2 -> fp16
        yield "s8", dict(m=m, n=c, c0=4 * c, has_residual=True, rowstats=True)  # ff.net.2 before an fp16 qkv
        yield "s8", dict(m=m, n=c, c0=4 * c, has_residual=True, out_s8=True)    # last ff.net.2 -> int8 proj_out
        yield "s8", dict(m=m, n=c, c0=c, has_residual=True)                     # proj_out
        yield "f16", dict(mode=0, m=m, n=8 * c, c0=c, geglu=True, ln=True, out_s8=True)     # fp16 GEGLU -> int8
        yield "f16", dict(mode=0, m=m, n=c, c0=4 * c, has_residual=True, out_s8=True)       # fp16 ff.net.2 -> int8


@pytest.mark.parametrize("model", sorted(MODELS))
def test_int8_linear_planner_gives_a_valid_plan_for_every_launch(model):
    from b200sd import lib

    lib.load()
    n = 0
    for kind, kw in _linear_launches(model):
        s = lib.describe_plan_s8_linear(**kw) if kind == "s8" else lib.describe_plan(**kw)
        p = _plan_fields(s)
        bn, sp, kb, kps, st = p["block_n"], p["splits"], p["kb_total"], p["kb_per_split"], p["stages"]
        assert bn in WIDTHS + ((16,) if kind == "s8" and not kw.get("out_s8") else ()), (kw, p)
        chunk = 128 if kind == "s8" else 64
        assert kb == math.ceil(kw["c0"] / chunk), (kw, p)  # each row zero padded to whole k-blocks (320 -> 384)
        per_stage = 128 * 128 + bn * 128
        assert 2 <= st <= 8 and st * per_stage + p["epi_smem"] + 1024 <= SMEM_LIMIT, (kw, p)
        assert st * per_stage >= 128 * (bn + 4) * 4, (kw, p)
        if p["cluster"]:
            assert sp in (2, 4, 8) and sp <= kb, (kw, p)
        else:
            assert sp * kps >= kb and (sp - 1) * kps < kb, (kw, p)
        if kw.get("out_s8"):
            assert p["variant"] == (7 if kw.get("geglu") else 6) and sp == 1, (kw, p)
        elif kw.get("geglu"):
            assert p["variant"] == 2 and sp == 1, (kw, p)
        elif kw.get("rowstats"):
            assert p["variant"] == 4 and sp == 1, (kw, p)
        else:
            assert p["variant"] in (0, 1, 4), (kw, p)
        assert p["staged"] == 0 and p["n_tiles"] * bn >= kw["n"], (kw, p)
        n += 1
    assert n >= 12


@pytest.mark.parametrize("field,kw", [
    ("mode", dict(mode=1)), ("a1", dict(c1=64)), ("act", dict(act=1)), ("out_f32", dict(out_f32=1)),
    ("bias_rows", dict(bias_rows=64)), ("halo", dict(halo=1)), ("upsample2x", dict(upsample2x=1)),
    ("gn_", dict(gn_groups=32)), ("cs_", dict(cs_partial=1)), ("ln_", dict(ln_parts=1)), ("a2 / a3", dict(c2=64)),
    ("pad_after_only", dict(pad_after_only=1)), ("c0", dict(c0=328)),
    ("out_s8_inv_scale", dict(out_s8_inv_scale=float("nan"))), ("out_s8_inv_scale", dict(out_s8_inv_scale=-1.0)),
    ("out_s8_inv_scale", dict(out_s8_inv_scale=1.0, split_k=2)),
    ("out_s8_inv_scale", dict(out_s8_inv_scale=1.0, rs_out=1)),
])
def test_int8_linear_planner_rejects_unsupported_fields_by_name(field, kw):
    from b200sd import lib

    lib.load()
    a = lib.GemmArgs()
    a.mode, a.m, a.n, a.c0 = 0, 512, 320, 320
    for k, v in kw.items():
        setattr(a, k, v)
    with pytest.raises(lib.B200SDError, match=re.escape(field)):
        lib.plan_ex_s8_linear(a)


@pytest.mark.parametrize("kw", [dict(mode=1, n_img=2, h=8, w=8), dict(out_f32=1), dict(n=336)])
def test_fp16_int8_output_rejects_unsupported_calls_by_name(kw):
    from b200sd import lib

    lib.load()
    a = lib.GemmArgs()
    a.mode, a.m, a.n, a.c0, a.out_s8_inv_scale = 0, 512, 320, 320, 0.5
    for k, v in kw.items():
        setattr(a, k, v)
    with pytest.raises(lib.B200SDError, match="out_s8_inv_scale"):
        lib.plan_ex(a)


def test_int8_linear_weight_tiling_pads_rows_to_whole_k_blocks():
    import torch
    from b200sd import lib

    g = torch.Generator().manual_seed(0)
    w = torch.randint(-127, 128, (96, 320), generator=g, dtype=torch.int8)
    t = lib.pack_tiled(w, 320, 0, 1, 32, chunk=128)
    assert t.shape == (3, 3, 32, 128)
    for nt in range(3):
        for j in range(3):
            lo, hi = 128 * j, min(128 * j + 128, 320)
            assert torch.equal(t[nt, j, :, : hi - lo], w[32 * nt:32 * nt + 32, lo:hi])
            assert not t[nt, j, :, hi - lo:].any()
