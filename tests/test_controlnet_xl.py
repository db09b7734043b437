"""CPU tests of ControlNet with SDXL: the SDXL ControlNet schema and restated ControlNet (controlnet_xl_oracle.py) against the fixtures of the
reference modules (tests/golden/make_golden_controlnet_xl.py), diffusers' guidance-window arithmetic, and the
ValueErrors of the pipeline's ControlNet arguments."""
import hashlib
import json
import os
import types

import sys

import numpy as np
import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import controlnet_xl_oracle as CX  # noqa: E402

from b200sd import config
from b200sd import pipeline as P
from b200sd import scheduler as S

GOLD = os.path.join(os.path.dirname(__file__), "golden")
FIXTURES = [("controlnet_tiny_xl", "TINY_XL_CONTROLNET", False), ("controlnet_sdxl", "SDXL_CONTROLNET", True)]


def _digest(shapes):
    lines = "\n".join(f"{k} {tuple(int(d) for d in v)}" for k, v in sorted(shapes.items()))
    return hashlib.sha256(lines.encode()).hexdigest()


def _fingerprint(sd):
    keys = sorted(sd.keys())
    picks = [keys[0], keys[len(keys) // 2], keys[-1]]
    return np.array([float(sd[k].double().sum()) for k in picks] + [float(len(keys))])


@pytest.mark.parametrize("name,cfg_name,fp16", FIXTURES)
def test_controlnet_xl_schema_matches_reference_modules(name, cfg_name, fp16):
    gold = np.load(os.path.join(GOLD, f"{name}.npz"))
    shapes = config.controlnet_param_shapes(getattr(config, cfg_name))
    assert _digest(shapes) == str(gold["schema"])
    assert "add_embedding.linear_1.weight" in shapes
    n = len(getattr(config, cfg_name)["block_out_channels"])
    depth = config._as_list(getattr(config, cfg_name)["transformer_layers_per_block"], n)[-1]
    assert f"mid_block.attentions.0.transformer_blocks.{depth - 1}.attn1.to_q.weight" in shapes
    assert f"mid_block.attentions.0.transformer_blocks.{depth}.attn1.to_q.weight" not in shapes


def test_sd_controlnet_schemas_unchanged():
    """Every SD 1.x / 2.x ControlNet has a depth-1 mid block and no add-embedding, as before."""
    for name in ("TINY_CONTROLNET", "SD21_CONTROLNET", "SD15_CONTROLNET", "TINY_SD1_CONTROLNET"):
        shapes = config.controlnet_param_shapes(getattr(config, name))
        assert not any(k.startswith("add_embedding") for k in shapes), name
        assert not any(k.startswith("mid_block.attentions.0.transformer_blocks.1.") for k in shapes), name


@pytest.mark.parametrize("name,cfg_name,fp16", FIXTURES)
def test_restated_controlnet_xl_matches_reference_golden(name, cfg_name, fp16):
    gold = np.load(os.path.join(GOLD, f"{name}.npz"))
    cfg = getattr(config, cfg_name)
    sd = config.random_state_dict(config.controlnet_param_shapes(cfg), seed=int(gold["weight_seed"]),
                                  dtype=torch.float16 if fp16 else torch.float32)
    assert np.allclose(_fingerprint(sd), gold["fingerprint"], rtol=1e-6), "weight generator drifted"
    size, st = int(gold["size"]), int(gold["stride"])
    pooled = cfg["projection_class_embeddings_input_dim"] - 6 * cfg["addition_time_embed_dim"]
    g = torch.Generator().manual_seed(int(gold["input_seed"]))
    x = torch.randn(2, 4, size, size, generator=g)
    ctx = torch.randn(2, cfg["cross_attention_dim"], 1, 77, generator=g)
    te = torch.randn(2, pooled, generator=g)
    cond = torch.rand(2, 3, 8 * size, 8 * size, generator=torch.Generator().manual_seed(int(gold["cond_seed"])))
    if fp16:
        x, ctx, te, cond = (v.half().float() for v in (x, ctx, te, cond))
    with torch.no_grad():
        outs = CX.controlnet_forward_xl(sd, cfg, x, torch.tensor([float(gold["timestep"])] * 2), ctx, cond,
                                        torch.from_numpy(gold["time_ids"]), te)
    assert len(outs) == len([k for k in gold.files if k.startswith("residual_")])
    for i, o in enumerate(outs):
        ref = torch.from_numpy(gold[f"residual_{i}"].astype(np.float32))
        err = float((o[:, :, ::st, ::st] - ref).abs().max())
        bar = 2e-3 * max(1.0, float(ref.abs().max())) if fp16 else 2e-5  # the fp16 fixture is stored in fp16
        assert err < bar, (name, i, err)


def _diffusers_keep(n, start, end):
    """diffusers 0.30's StableDiffusionXLControlNetPipeline: controlnet_keep."""
    keeps = []
    for i in range(n):
        k = [1.0 - float(i / n < s or (i + 1) / n > e) for s, e in zip(start, end)]
        keeps.append(k)
    return keeps


def _img2img_steps(n, strength):
    sched = S.make_scheduler("DDIM", n)
    return len(list(sched.plan(start=sched.start_step(strength))))


@pytest.mark.parametrize("n,start,end", [
    (20, [0.0], [1.0]), (20, [0.0, 0.0], [1.0, 0.5]), (20, [0.1], [0.9]), (7, [0.0, 0.3], [0.5, 1.0]),
    (3, [0.5], [1.0]), (1, [0.0], [1.0]), (1, [0.5], [1.0]), (50, [0.2, 0.0, 0.7], [0.8, 0.35, 1.0]),
    (_img2img_steps(20, 0.5), [0.0, 0.25], [0.6, 1.0]), (_img2img_steps(30, 0.75), [0.1], [0.45]),
])
def test_controlnet_keep_matches_diffusers(n, start, end):
    keep = P.controlnet_keep(n, start, end)
    ref = _diffusers_keep(n, start, end)
    assert len(keep) == n
    for i in range(n):
        assert keep[i] == tuple(k for k, v in enumerate(ref[i]) if v == 1.0), (i, keep[i], ref[i])


def test_img2img_keep_counts_executed_steps():
    n = _img2img_steps(20, 0.5)
    assert n == 10
    assert P.controlnet_keep(n, [0.0], [0.5]) == [(0,)] * 5 + [()] * 5


def test_controlnet_arguments_errors():
    assert P.controlnet_arguments(2, 0.5) == ([0.5, 0.5], [0.0, 0.0], [1.0, 1.0])
    assert P.controlnet_arguments(2, [0.7, 0.3], 0.0, [1.0, 0.5]) == ([0.7, 0.3], [0.0, 0.0], [1.0, 0.5])
    with pytest.raises(ValueError, match="controlnet_conditioning_scale has 3 values for 2"):
        P.controlnet_arguments(2, [1.0, 1.0, 1.0])
    with pytest.raises(ValueError, match="control_guidance_start has 1 values for 2"):
        P.controlnet_arguments(2, 1.0, [0.0])
    with pytest.raises(ValueError, match="control_guidance_end has 3 values"):
        P.controlnet_arguments(2, 1.0, 0.0, [1.0, 1.0, 1.0])
    for start, end in ((0.5, 0.5), (0.6, 0.4), (-0.1, 1.0), (0.0, 1.5)):
        with pytest.raises(ValueError, match="control_guidance_start / control_guidance_end"):
            P.controlnet_arguments(1, 1.0, start, end)
    for bad in (float("nan"), float("inf"), [1.0, float("-inf")]):
        with pytest.raises(ValueError, match="controlnet_conditioning_scale must be finite"):
            P.controlnet_arguments(2, bad)
    with pytest.raises(ValueError, match="guess_mode"):
        P.controlnet_arguments(1, guess_mode=True)


def test_call_refuses_guess_mode():
    pipe = P.B200StableDiffusionPipeline.__new__(P.B200StableDiffusionPipeline)
    with pytest.raises(ValueError, match="guess_mode"):
        pipe("a cat", guess_mode=True)


@pytest.mark.parametrize("field,value", [
    ("cross_attention_dim", 1024), ("block_out_channels", (320, 640, 640)),
    ("down_block_types", ("CrossAttnDownBlock2D", "CrossAttnDownBlock2D", "DownBlock2D")), ("layers_per_block", 1),
    ("addition_embed_type", None), ("projection_class_embeddings_input_dim", 2560),
])
def test_mismatched_controlnet_is_refused(field, value):
    config.check_controlnet_matches_unet(config.SDXL_BASE_UNET, config.SDXL_CONTROLNET)
    with pytest.raises(ValueError, match=field):
        config.check_controlnet_matches_unet(config.SDXL_BASE_UNET, dict(config.SDXL_CONTROLNET, **{field: value}))
    # the pipeline constructor runs the same check on its ControlNets
    unet = types.SimpleNamespace(use_cuda_graph=False, device="cpu",
                                 engine=types.SimpleNamespace(support_controlnet=True, cfg=config.SDXL_BASE_UNET))
    net = types.SimpleNamespace(engine=types.SimpleNamespace(cfg=dict(config.SDXL_CONTROLNET, **{field: value})))
    with pytest.raises(ValueError, match=field):
        P.B200StableDiffusionPipeline(unet, None, controlnet=[net], xl=True)


def test_sd_controlnets_match_their_unets():
    for u, c in ((config.SD21_BASE_UNET, config.SD21_CONTROLNET), (config.SD15_UNET, config.SD15_CONTROLNET),
                 (config.TINY_UNET, config.TINY_CONTROLNET), (config.TINY_SD1_UNET, config.TINY_SD1_CONTROLNET),
                 (config.TINY_XL_UNET, config.TINY_XL_CONTROLNET), (config.SDXL_BASE_UNET, config.SDXL_CONTROLNET)):
        config.check_controlnet_matches_unet(u, c)
    with pytest.raises(ValueError, match="cross_attention_dim"):
        config.check_controlnet_matches_unet(config.SDXL_BASE_UNET, config.SD21_CONTROLNET)


def test_global_pool_controlnet_is_refused():
    with pytest.raises(ValueError, match="global_pool_conditions"):
        config.check_controlnet_matches_unet(config.SDXL_BASE_UNET, dict(config.SDXL_CONTROLNET,
                                                                         global_pool_conditions=True))


def test_controlnet_with_refiner_is_refused(tmp_path):
    unet = types.SimpleNamespace(use_cuda_graph=False, device="cpu",
                                 engine=types.SimpleNamespace(support_controlnet=True, cfg=config.SDXL_BASE_UNET))
    net = types.SimpleNamespace(engine=types.SimpleNamespace(cfg=config.SDXL_CONTROLNET))
    with pytest.raises(ValueError, match="refiner"):
        P.B200StableDiffusionPipeline(unet, None, controlnet=[net], xl=True, unet_refiner=object())
    # from_pretrained refuses the combination before reading any weights
    for d, cfg in (("base/unet", config.SDXL_BASE_UNET), ("base/vae", config.SDXL_VAE), ("cn", config.SDXL_CONTROLNET)):
        os.makedirs(tmp_path / d)
        (tmp_path / d / "config.json").write_text(json.dumps({k: (list(v) if isinstance(v, tuple) else v)
                                                              for k, v in cfg.items()}))
    with pytest.raises(ValueError, match="refiner"):
        P.B200StableDiffusionPipeline.from_pretrained(str(tmp_path / "base"), controlnet_dirs=[str(tmp_path / "cn")],
                                                      refiner_dir=str(tmp_path / "refiner"))
    (tmp_path / "cn" / "config.json").write_text(json.dumps(dict(
        {k: (list(v) if isinstance(v, tuple) else v) for k, v in config.SDXL_CONTROLNET.items()},
        layers_per_block=1)))
    with pytest.raises(ValueError, match="layers_per_block"):
        P.B200StableDiffusionPipeline.from_pretrained(str(tmp_path / "base"), controlnet_dirs=[str(tmp_path / "cn")])
