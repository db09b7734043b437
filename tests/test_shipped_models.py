"""Host-only tests of the shipped-model list both per-launch replays run (model_cases.SHIPPED) and of the SDXL refiner's
configuration."""
import os
import re
import sys
import types

import pytest

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import model_cases as MC  # noqa: E402
from b200sd import config as C  # noqa: E402
from b200sd import lib as L  # noqa: E402

# The published stabilityai/stable-diffusion-xl-refiner-1.0 unet/config.json, as the pipeline reads it
# (checkpoint.read_config): no num_time_ids key.
REFINER_JSON = dict(
    act_fn="silu", addition_embed_type="text_time", addition_embed_type_num_heads=64, addition_time_embed_dim=256,
    attention_head_dim=(6, 12, 24, 24), block_out_channels=(384, 768, 1536, 1536), center_input_sample=False,
    cross_attention_dim=1280, down_block_types=("DownBlock2D", "CrossAttnDownBlock2D", "CrossAttnDownBlock2D",
                                                "DownBlock2D"),
    downsample_padding=1, flip_sin_to_cos=True, freq_shift=0, in_channels=4, layers_per_block=2, mid_block_scale_factor=1,
    norm_eps=1e-05, norm_num_groups=32, out_channels=4, projection_class_embeddings_input_dim=2560, sample_size=128,
    transformer_layers_per_block=4, up_block_types=("UpBlock2D", "CrossAttnUpBlock2D", "CrossAttnUpBlock2D", "UpBlock2D"),
    upcast_attention=False, use_linear_projection=True)


def test_refiner_config_matches_published():
    for k, v in REFINER_JSON.items():
        if k in C.SDXL_REFINER_UNET:
            assert C.SDXL_REFINER_UNET[k] == v, k


def test_refiner_head_dims_and_add_embedding_width():
    cfg = C.SDXL_REFINER_UNET
    for ch, heads in zip(cfg["block_out_channels"], cfg["attention_head_dim"]):
        assert ch % heads == 0 and ch // heads in L.ATTENTION_HEAD_DIMS, (ch, heads)
    assert cfg["num_time_ids"] * cfg["addition_time_embed_dim"] + C.SDXL_POOLED_DIM == \
        cfg["projection_class_embeddings_input_dim"]


def test_num_time_ids_from_a_config_without_the_count():
    """A diffusers config names only add_embedding's width: 5 time ids for the refiner, 6 for SDXL-base."""
    assert C.num_time_ids(REFINER_JSON) == 5
    assert C.num_time_ids({k: v for k, v in C.SDXL_BASE_UNET.items() if k != "num_time_ids"}) == 6
    assert C.num_time_ids(C.SDXL_REFINER_UNET) == 5
    assert C.num_time_ids(C.TINY_XL_UNET, pooled_dim=64) == 6
    with pytest.raises(ValueError):
        C.num_time_ids(dict(REFINER_JSON, projection_class_embeddings_input_dim=2600))


def test_refiner_param_schema():
    sh = C.unet_param_shapes(C.SDXL_REFINER_UNET)
    assert sh["conv_in.weight"] == (384, 4, 3, 3)
    assert sh["time_embedding.linear_1.weight"] == (1536, 384, 1, 1)
    assert sh["add_embedding.linear_1.weight"] == (1536, 2560, 1, 1)
    # cross-attention levels 1 and 2 and the mid block, each with depth-4 transformers on 1280-wide text states
    for p, c in (("down_blocks.1.attentions.1", 768), ("down_blocks.2.attentions.0", 1536),
                 ("mid_block.attentions.0", 1536), ("up_blocks.1.attentions.2", 1536), ("up_blocks.2.attentions.0", 768)):
        assert sh[f"{p}.transformer_blocks.3.attn2.to_k.weight"] == (c, 1280, 1, 1), p
        assert f"{p}.transformer_blocks.4.attn1.to_q.weight" not in sh, p
    assert not any(k.startswith(("down_blocks.0.attentions", "down_blocks.3.attentions", "up_blocks.0.attentions",
                                 "up_blocks.3.attentions")) for k in sh)
    # the skip concatenations: 1536 + 1536 = 3072, 1536 + 768 = 2304, 768 + 384 = 1152
    assert sh["up_blocks.0.resnets.0.norm1.weight"] == (3072,)
    assert sh["up_blocks.1.resnets.2.norm1.weight"] == (2304,)
    assert sh["up_blocks.3.resnets.0.norm1.weight"] == (1152,)
    assert sh["up_blocks.3.resnets.2.conv1.weight"] == (384, 768, 3, 3)
    assert sh["conv_out.weight"] == (4, 384, 3, 3)


def test_shipped_list_covers_every_path():
    assert len(set(MC.SHIPPED)) == len(MC.SHIPPED)
    assert all(MC.SHIPPED_PATHS[n].strip() for n in MC.SHIPPED)
    for name in ("sdxl_1024_b2", "sdxl_refiner_1024_b2", "sdxl_refiner_768_b2", "vae_decoder_768", "vae_decoder_bf16_768",
                 "vae_encoder_512", "vae_encoder_768", "vae_encoder_bf16_1024", "controlnet_sd15", "controlnet_sd21_768",
                 "sd21_b2", "sd21_b16", "sd15_b2", "sdxl_768_b2", "controlnet_sd21", "vae_decoder", "openclip_h", "clip_l",
                 "sd21_768_b2", "vae_decoder_bf16", "vae_encoder_bf16", "openclip_bigg", "sd15_512x768_b2",
                 "sd15_768x512_b2", "sd21_576x576_b2", "sdxl_768x1344_b2", "sdxl_1216x832_b2",
                 "sdxl_refiner_768x1344_b2", "controlnet_sd15_512x768", "vae_decoder_512x768", "vae_decoder_bf16_768x1344", "vae_encoder_768x512",
                 "vae_encoder_bf16_1216x832"):
        assert name in MC.SHIPPED, name


def test_both_replays_run_the_shipped_list():
    import test_gemm_plans_gpu as GP
    import test_op_launches_gpu as OP

    assert set(MC.SHIPPED) <= set(GP.MODELS) and set(MC.SHIPPED) <= set(OP.MODELS)
    assert set(GP.MODELS) - set(MC.SHIPPED) == {"sd21_b2_fused", "sd21_b2_halo_tma", "sd15_512x768_b2_fused",
                                                "sd15_512x768_b2_halo_tma"}
    assert set(OP.MODELS) - set(MC.SHIPPED) == {"sd21_b2_fused2", "sd15_512x768_b2_fused2"}
    # every non-square or off-grid shipped name has the shapes it exists for asserted in the op replay
    assert {n for n in MC.SHIPPED if re.search(r"_\d+x\d+", n)} == set(OP.NON_SQUARE_SHAPES)


# latents of every name with an explicit pixel size, and of the square names as they were before sizes were parsed
LATENT_HW = {
    "sd15_512x768_b2": (64, 96), "sd15_768x512_b2": (96, 64), "sd21_576x576_b2": (72, 72),
    "sdxl_768x1344_b2": (96, 168), "sdxl_1216x832_b2": (152, 104), "sdxl_refiner_768x1344_b2": (96, 168),
    "controlnet_sd15_512x768": (64, 96), "vae_decoder_512x768": (64, 96), "vae_decoder_bf16_768x1344": (96, 168),
    "vae_encoder_768x512": (96, 64), "vae_encoder_bf16_1216x832": (152, 104),
    "sd21_b2": (64, 64), "sd21_b16": (64, 64), "sd15_b2": (64, 64), "sd21_768_b2": (96, 96), "sdxl_768_b2": (96, 96),
    "sdxl_1024_b2": (128, 128), "sdxl_refiner_1024_b2": (128, 128), "sdxl_refiner_768_b2": (96, 96),
    "controlnet_sd21": (64, 64), "controlnet_sd15": (64, 64), "controlnet_sd21_768": (96, 96), "vae_decoder": (64, 64),
    "vae_decoder_768": (96, 96), "vae_decoder_bf16": (128, 128), "vae_decoder_bf16_768": (96, 96),
    "vae_encoder_512": (64, 64), "vae_encoder_768": (96, 96), "vae_encoder_bf16": (64, 64),
    "vae_encoder_bf16_1024": (128, 128),
}


def test_every_name_maps_to_its_size():
    """An explicit <height>x<width> is parsed before the "768" / "1024" substrings (sd15_512x768_b2 is 64x96, not 96^2),
    and the square names keep the geometry they had."""
    assert set(LATENT_HW) == {n for n in MC.SHIPPED if not n.startswith(("openclip", "clip"))}
    for name, hw in LATENT_HW.items():
        assert MC.latent_hw(name) == hw, name
    for name in ("sd15_512x768_b2_fused", "sd15_512x768_b2_halo_tma", "sd15_512x768_b2_fused2"):
        assert MC.latent_hw(name) == (64, 96), name
    assert MC.latent_hw("sd21_b2_fused") == (64, 64)


def _model_cfg(name):
    if name.startswith("controlnet"):
        return C.SD15_CONTROLNET if name.startswith("controlnet_sd15") else C.SD21_CONTROLNET
    if name.startswith("sdxl_refiner"):
        return C.SDXL_REFINER_UNET
    return C.SD21_UNET if name.startswith("sd21_768") else {"sd21": C.SD21_BASE_UNET, "sd15": C.SD15_UNET,
                                                             "sdxl": C.SDXL_BASE_UNET}[name[:4]]


@pytest.mark.parametrize("name", [n for n in MC.SHIPPED if n.startswith(("sd", "controlnet"))])
def test_shipped_unet_sizes_halve_exactly(name):
    """Every down-sampler of a shipped UNet / ControlNet halves its map exactly: the latents divide by
    2^(levels - 1), so the constructor's size check accepts them."""
    cfg = _model_cfg(name)
    h, w = MC.latent_hw(name)
    levels = len(cfg["block_out_channels"])
    assert h % 2 ** (levels - 1) == 0 and w % 2 ** (levels - 1) == 0, (name, h, w)
    C.check_latent_size(cfg, h, w)


def test_latent_multiple():
    """64 pixels for SD 1.x / 2.x, their ControlNets and the refiner (four levels), 32 for SDXL-base (three); the check
    names the pixel multiple and rejects either dimension alone."""
    for cfg in (C.SD21_BASE_UNET, C.SD21_UNET, C.SD15_UNET, C.SDXL_REFINER_UNET, C.SD21_CONTROLNET, C.SD15_CONTROLNET):
        assert C.latent_multiple(cfg) == 8
    assert C.latent_multiple(C.SDXL_BASE_UNET) == 4
    assert C.latent_multiple(C.TINY_UNET) == 4 and C.latent_multiple(C.TINY_XL_UNET) == 2
    C.check_latent_size(C.SD15_UNET, 64, 96)
    C.check_latent_size(C.SDXL_BASE_UNET, 100, 132)  # 800x1056: SDXL-base takes multiples of 32 pixels
    for h, w in ((68, 68), (64, 68), (68, 64), (72, 76)):  # 544^2 halves 68 -> 34 -> 17 and cannot go on
        with pytest.raises(ValueError, match="multiples of 64 pixels"):
            C.check_latent_size(C.SD15_UNET, h, w)
    with pytest.raises(ValueError, match="multiples of 64 pixels"):
        C.check_latent_size(C.SDXL_REFINER_UNET, 96, 164)
    with pytest.raises(ValueError, match="multiples of 32 pixels"):
        C.check_latent_size(C.SDXL_BASE_UNET, 96, 166)


@pytest.mark.parametrize("nid,h,want", [(6, 128, [1024.0, 1024.0, 0.0, 0.0, 1024.0, 1024.0]),
                                        (5, 96, [768.0, 768.0, 0.0, 0.0, 6.0])])
def test_model_inputs_time_ids(nid, h, want):
    """The time ids are as wide as the model declares, and hold its image size (and the refiner's aesthetic score)."""
    import numpy as np

    m = types.SimpleNamespace(h=h, w=h, expected_inputs={"time_ids": {"shape": (2, nid), "dtype": np.float16}})
    ids = MC.model_inputs(m, seed=0)["time_ids"]
    assert ids.shape == (2, nid) and ids.tolist() == [want, want]
