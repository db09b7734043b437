"""Host-only tests of the shipped-model list both per-launch replays run (model_cases.SHIPPED) and of the SDXL refiner's
configuration."""
import os
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
                 "sd21_768_b2", "vae_decoder_bf16", "vae_encoder_bf16", "openclip_bigg"):
        assert name in MC.SHIPPED, name


def test_both_replays_run_the_shipped_list():
    import test_gemm_plans_gpu as GP
    import test_op_launches_gpu as OP

    assert set(MC.SHIPPED) <= set(GP.MODELS) and set(MC.SHIPPED) <= set(OP.MODELS)
    assert set(GP.MODELS) - set(MC.SHIPPED) == {"sd21_b2_fused", "sd21_b2_halo_tma"}
    assert set(OP.MODELS) - set(MC.SHIPPED) == {"sd21_b2_fused2"}


@pytest.mark.parametrize("nid,h,want", [(6, 128, [1024.0, 1024.0, 0.0, 0.0, 1024.0, 1024.0]),
                                        (5, 96, [768.0, 768.0, 0.0, 0.0, 6.0])])
def test_model_inputs_time_ids(nid, h, want):
    """The time ids are as wide as the model declares, and hold its image size (and the refiner's aesthetic score)."""
    import numpy as np

    m = types.SimpleNamespace(h=h, w=h, expected_inputs={"time_ids": {"shape": (2, nid), "dtype": np.float16}})
    ids = MC.model_inputs(m, seed=0)["time_ids"]
    assert ids.shape == (2, nid) and ids.tolist() == [want, want]
