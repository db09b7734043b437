"""Weight palettization on the host (no GPU): eligible layers, palette fitting, index packing and recipe parsing."""
import json
import math

import pytest
import torch

from b200sd import config as C
from b200sd import palettization as Pz


def test_eligible_layers_follow_the_size_rule():
    for cfg in (C.SD21_BASE_UNET, C.SD15_UNET, C.SDXL_BASE_UNET, C.TINY_UNET):
        layers = Pz.palettizable_layers(cfg)
        shapes = C.unet_param_shapes(cfg)
        assert layers
        for name, numel in layers.items():
            assert numel == math.prod(shapes[name + ".weight"]) > 100_000
        small = [k for k, s in shapes.items() if k.endswith(".weight") and len(s) in (2, 4) and math.prod(s) <= 100_000]
        assert not any(k[:-7] in layers for k in small)
    sd21 = Pz.palettizable_layers(C.SD21_BASE_UNET)
    assert "down_blocks.0.attentions.0.transformer_blocks.0.attn1.to_q" in sd21
    assert "conv_in" not in sd21 and "conv_out" not in sd21


@pytest.mark.parametrize("key,cfg", [("sd21_base", C.SD21_BASE_UNET), ("sd15", C.SD15_UNET), ("sdxl_base", C.SDXL_BASE_UNET)])
def test_eligible_layers_equal_the_reference_module_lists(key, cfg):
    """tests/golden/palettizable_layers.json holds the reference UNet's module names (the recipe JSON keys) that pass
    its get_palettizable_modules rule (make_golden_palettization.py)."""
    import os

    with open(os.path.join(os.path.dirname(__file__), "golden", "palettizable_layers.json")) as f:
        golden = json.load(f)[key]
    assert Pz.palettizable_layers(cfg) == golden


def test_lut_plans_fit_where_the_fp16_plans_do():
    """Wide tiles with a residual tile in shared memory at 1 / 2 bits need more packed-index slots than pipeline
    stages to park the accumulator tile (host-only planning, no GPU)."""
    from b200sd import lib as L

    for nbits in Pz.NBITS:
        for m, n, c in ((32768, 1280, 1280), (8192, 1280, 1280), (512, 640, 640), (2048, 320, 320)):
            args = L.GemmArgs()
            args.mode, args.m, args.n, args.c0 = 0, m, n, c
            args.bias, args.residual = 16, 16
            fp16 = L.describe_plan(0, m=m, n=n, c0=c, has_bias=True, has_residual=True)
            pw = Pz.PalettizedWeight(torch.zeros(n, Pz.row_bytes(c, nbits), dtype=torch.uint8),
                                     torch.zeros(3, 256, dtype=torch.float16), nbits, c)
            desc = L.describe_plan_lut(args, pw)
            for key in ("block_n", "splits", "kb_per_split", "cluster"):
                f = fp16.split(f"{key}=")[1].split()[0]
                assert desc.split(f"{key}=")[1].split()[0] == f, (nbits, m, desc, fp16)


def test_fit_is_deterministic_and_exact_on_few_values():
    g = torch.Generator().manual_seed(0)
    w = torch.randn(320, 640, generator=g)
    for nbits in Pz.NBITS:
        a = Pz.fit_palette(w, nbits)
        b = Pz.fit_palette(w.clone(), nbits)
        assert torch.equal(a[0], b[0]) and torch.equal(a[1], b[1])
        assert a[0].numel() == 2 ** nbits and a[0].dtype == torch.float16
    vals = torch.tensor([-0.5, 0.0, 0.25, 1.5])
    w4 = vals[torch.randint(0, 4, (128, 64), generator=g)]
    lut, idx = Pz.fit_palette(w4, 2)
    assert torch.equal(Pz.decode(lut, idx).float(), w4)
    lut, idx = Pz.fit_palette(w4, 4)  # more entries than values
    assert torch.equal(Pz.decode(lut, idx).float(), w4)


@pytest.mark.parametrize("nbits", Pz.NBITS)
def test_each_index_is_the_nearest_entry(nbits):
    w = torch.randn(256, 256, generator=torch.Generator().manual_seed(nbits))
    lut, idx = Pz.fit_palette(w, nbits)
    wv = w.half().double().reshape(-1, 1)
    d = (wv - lut.double()[None, :]).abs()
    best = d.min(1).values
    chosen = d.gather(1, idx.reshape(-1, 1).long()).squeeze(1)
    assert torch.equal(chosen, best)
    # ties go to the lower index: no lower entry is as near
    lower = (d <= best[:, None]) & (torch.arange(lut.numel())[None, :] < idx.reshape(-1, 1).long())
    assert not lower.any()


@pytest.mark.parametrize("dist", ["gauss", "laplace"])
@pytest.mark.parametrize("shape", [(320, 320), (1280, 11520 // 9, 3, 3), (640, 2048)])
@pytest.mark.parametrize("nbits", Pz.NBITS)
def test_palette_mse_beats_a_uniform_grid(dist, shape, nbits):
    g = torch.Generator().manual_seed(nbits * 10 + len(shape) + (dist == "laplace"))
    w = torch.randn(*shape, generator=g) * 0.02
    if dist == "laplace":
        u = (torch.rand(*shape, generator=g) - 0.5) * 0.999
        w = -0.02 * torch.sign(u) * torch.log1p(-2 * u.abs())
    wh = w.half().double()
    lut, idx = Pz.fit_palette(w, nbits)
    mse = ((Pz.decode(lut, idx).double() - wh) ** 2).mean()
    lo, hi = wh.min(), wh.max()
    k = 2 ** nbits
    step = (hi - lo) / (k - 1)
    uni = torch.round((wh - lo) / step) * step + lo
    mse_u = ((uni - wh) ** 2).mean()
    assert mse <= mse_u


@pytest.mark.parametrize("nbits", Pz.NBITS)
def test_pack_round_trip(nbits):
    g = torch.Generator().manual_seed(nbits)
    idx = torch.randint(0, 2 ** nbits, (48, 9 * 64), generator=g).to(torch.uint8)
    packed = Pz.pack_indices(idx, nbits)
    assert packed.dtype == torch.uint8 and packed.shape == (48, Pz.row_bytes(9 * 64, nbits))
    assert packed.shape[1] % 16 == 0
    assert torch.equal(Pz.unpack_indices(packed, nbits, 9 * 64), idx)
    # little-endian bit stream: index k at bits [k * nbits, (k + 1) * nbits)
    row = packed[0].tolist()
    stream = sum(b << (8 * i) for i, b in enumerate(row))
    for k in range(0, 9 * 64, 37):
        assert (stream >> (k * nbits)) & ((1 << nbits) - 1) == int(idx[0, k])


def test_segmented_weight_decodes_each_segment_with_its_palette():
    g = torch.Generator().manual_seed(3)
    ws = [torch.randn(64, 128, generator=g) for _ in range(3)]
    fits = [Pz.fit_palette(w, n) for w, n in zip(ws, (2, 4, 6))]
    gamma = torch.rand(128, generator=g) + 0.5
    pw = Pz.palettized([(l, i, n) for (l, i), n in zip(fits, (2, 4, 6))], kscale=gamma)
    assert pw.nbits == 6 and pw.nominal == (2, 4, 6) and pw.seg_ends == (64, 128)
    ref = torch.cat([Pz.decode(l, i) for l, i in fits], 0)
    assert torch.equal(pw.decoded(), (ref.float() * gamma[None, :]).half())


def test_recipe_forms(tmp_path):
    cfg = C.SD21_BASE_UNET
    layers = Pz.palettizable_layers(cfg)
    assert Pz.as_recipe(None, cfg) is None
    assert Pz.as_recipe(4, cfg) == {k: 4 for k in layers}
    assert Pz.as_recipe(16, cfg) == {}
    names = list(layers)
    rec = {names[0]: 6, names[1]: 16, names[2]: 1}
    assert Pz.as_recipe(rec, cfg) == {names[0]: 6, names[2]: 1}
    path = tmp_path / "pre.json"
    path.write_text(json.dumps({"model_version": "stabilityai/stable-diffusion-2-1-base",
                                "baselines": {"original": 40.0, "recipe_4.50_bit_mixedpalette": 30.1},
                                "recipes": {"recipe_4.50_bit_mixedpalette": rec}}))
    assert Pz.as_recipe((str(path), "recipe_4.50_bit_mixedpalette"), cfg) == {names[0]: 6, names[2]: 1}
    assert Pz.nominal_bits({names[0]: 6}, cfg) < 16


def test_malformed_recipes_raise(tmp_path):
    cfg = C.SD21_BASE_UNET
    name = next(iter(Pz.palettizable_layers(cfg)))
    with pytest.raises(ValueError, match="unknown layer down_blocks.9.nothing"):
        Pz.as_recipe({"down_blocks.9.nothing": 4}, cfg)
    with pytest.raises(ValueError, match="conv_in is not eligible"):
        Pz.as_recipe({"conv_in": 4}, cfg)
    with pytest.raises(ValueError, match=f"{name}: nbits=3"):
        Pz.as_recipe({name: 3}, cfg)
    with pytest.raises(ValueError, match="nbits=5"):
        Pz.as_recipe(5, cfg)
    path = tmp_path / "pre.json"
    path.write_text(json.dumps({"recipes": {"a": {}, "b": {}}}))
    with pytest.raises(ValueError, match=r"'c' is not in .*available recipes: \['a', 'b'\]"):
        Pz.as_recipe((str(path), "c"), cfg)


def test_decoded_state_dict_replaces_only_recipe_weights():
    cfg = C.TINY_UNET
    sd = C.random_state_dict(C.unet_param_shapes(cfg), seed=1)
    rec = Pz.as_recipe(2, cfg)
    dec = Pz.decoded_state_dict(sd, rec)
    for k, v in sd.items():
        if k.endswith(".weight") and k[:-7] in rec:
            assert dec[k].dtype == torch.float16 and dec[k].shape == v.shape
            assert torch.unique(dec[k]).numel() <= 4
        else:
            assert dec[k] is v
