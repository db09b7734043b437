"""Model configurations and parameter schemas for the b200sd hot path.

The configs mirror the keyword arguments of the reference constructors
(``python_coreml_stable_diffusion/unet.py:800-832`` ``UNet2DConditionModel.__init__``;
``controlnet.py:52-70``) and the diffusers ``AutoencoderKL`` config read by
``torch2coreml.py:548-642``.  Parameter names are the diffusers state-dict keys the reference
loads (``unet.py:121-146`` hooks).
"""
from __future__ import annotations

from collections import OrderedDict

import torch

SD21_BASE_UNET = dict(
    sample_size=64, in_channels=4, out_channels=4,
    down_block_types=("CrossAttnDownBlock2D", "CrossAttnDownBlock2D", "CrossAttnDownBlock2D", "DownBlock2D"),
    up_block_types=("UpBlock2D", "CrossAttnUpBlock2D", "CrossAttnUpBlock2D", "CrossAttnUpBlock2D"),
    block_out_channels=(320, 640, 1280, 1280), layers_per_block=2,
    attention_head_dim=(5, 10, 20, 20),  # == number of heads (unet.py:194-197)
    cross_attention_dim=1024, norm_num_groups=32, norm_eps=1e-5,
    flip_sin_to_cos=True, freq_shift=0, transformer_layers_per_block=1,
)

# SD 2.0 / 2.1 768-v (stabilityai/stable-diffusion-2-1): the SD-2.1-base UNet trained at 768x768 (96x96 latents) as a
# v-prediction model.  Its diffusers config also sets upcast_attention and use_linear_projection: the attention kernels
# already accumulate QK^T and the softmax in fp32, which is what upcast_attention asks for, and the [out, in] weights of a
# linear proj_in / proj_out are what the engine makes of a 1x1 convolution's anyway (checkpoint.check_state_dict accepts
# either shape).
SD21_UNET = dict(SD21_BASE_UNET, sample_size=96)

# SD 1.4 / 1.5 (CompVis/stable-diffusion-v1-4, the reference's default model): SD-2.1-base with 8 heads in every block
# (head dims 40 / 80 / 160) and the 768-wide CLIP ViT-L/14 text states; the reference constructor's defaults
# (unet.py:826-828).  859,520,964 parameters.
SD15_UNET = dict(SD21_BASE_UNET, attention_head_dim=8, cross_attention_dim=768)

SDXL_BASE_UNET = dict(
    sample_size=128, in_channels=4, out_channels=4,
    down_block_types=("DownBlock2D", "CrossAttnDownBlock2D", "CrossAttnDownBlock2D"),
    up_block_types=("CrossAttnUpBlock2D", "CrossAttnUpBlock2D", "UpBlock2D"),
    block_out_channels=(320, 640, 1280), layers_per_block=2,
    attention_head_dim=(5, 10, 20), cross_attention_dim=2048,
    norm_num_groups=32, norm_eps=1e-5, flip_sin_to_cos=True, freq_shift=0,
    transformer_layers_per_block=(1, 2, 10),
    addition_embed_type="text_time", addition_time_embed_dim=256,
    projection_class_embeddings_input_dim=2816,
)

# SDXL refiner (stabilityai/stable-diffusion-xl-refiner-1.0 unet/config.json): four levels of 384 / 768 / 1536 / 1536
# channels, 6 / 12 / 24 / 24 heads of 64, depth-4 transformers, conditioned on OpenCLIP bigG alone (1280-wide states).
# Its time ids are five (original size, crop, aesthetic score): 5 x 256 sinusoids + the 1280-wide pooled embedding =
# 2560 inputs of add_embedding.  The published file does not name that count; num_time_ids() derives it.
SDXL_REFINER_UNET = dict(
    sample_size=128, in_channels=4, out_channels=4,
    down_block_types=("DownBlock2D", "CrossAttnDownBlock2D", "CrossAttnDownBlock2D", "DownBlock2D"),
    up_block_types=("UpBlock2D", "CrossAttnUpBlock2D", "CrossAttnUpBlock2D", "UpBlock2D"),
    block_out_channels=(384, 768, 1536, 1536), layers_per_block=2,
    attention_head_dim=(6, 12, 24, 24), cross_attention_dim=1280,
    norm_num_groups=32, norm_eps=1e-5, flip_sin_to_cos=True, freq_shift=0,
    transformer_layers_per_block=4,
    addition_embed_type="text_time", addition_time_embed_dim=256,
    projection_class_embeddings_input_dim=2560, num_time_ids=5,
)

# width of the pooled text embedding an SDXL UNet's add_embedding reads next to the time ids (OpenCLIP bigG's
# projection_dim, the second text encoder of SDXL-base and the refiner's only one)
SDXL_POOLED_DIM = 1280


def num_time_ids(cfg, pooled_dim=SDXL_POOLED_DIM) -> int:
    """How many time ids a `text_time` UNet takes: cfg["num_time_ids"] when given, else what the pooled embedding
    leaves of add_embedding's input, (projection_class_embeddings_input_dim - pooled_dim) / addition_time_embed_dim:
    6 for SDXL-base (2816), 5 for the refiner (2560).  A diffusers config.json names only the total."""
    if cfg.get("num_time_ids"):
        return int(cfg["num_time_ids"])
    rest = cfg["projection_class_embeddings_input_dim"] - pooled_dim
    ate = cfg["addition_time_embed_dim"]
    if rest <= 0 or rest % ate:
        raise ValueError(f"projection_class_embeddings_input_dim {cfg['projection_class_embeddings_input_dim']} is not "
                         f"a {pooled_dim}-wide pooled embedding plus a whole number of {ate}-wide time ids")
    return rest // ate


def latent_multiple(cfg) -> int:
    """What the latent height and width of a UNet or ControlNet must be a multiple of: each of its
    len(block_out_channels) - 1 down-samplers halves the map (stride 2), and the up-samplers double it back onto the
    skip connections, so every halving must be exact.  8 (images of a multiple of 64 pixels) for SD 1.x / 2.x and the
    SDXL refiner, 4 (32 pixels) for SDXL-base."""
    return 2 ** (len(cfg["block_out_channels"]) - 1)


def check_latent_size(cfg, height, width, what="UNet"):
    """ValueError unless latents of height x width can be halved by every down-sampler of the model
    (latent_multiple)."""
    m = latent_multiple(cfg)
    if height % m or width % m:
        raise ValueError(f"{what}: latents of {height}x{width} ({8 * height}x{8 * width} pixels) cannot be halved "
                         f"{len(cfg['block_out_channels']) - 1} times; height and width must be multiples of {8 * m} "
                         f"pixels ({m} latent pixels) for this model")


# small config for fast CPU/GPU parity tests (same topology, d_head = 64)
TINY_UNET = dict(
    sample_size=16, in_channels=4, out_channels=4,
    down_block_types=("CrossAttnDownBlock2D", "CrossAttnDownBlock2D", "DownBlock2D"),
    up_block_types=("UpBlock2D", "CrossAttnUpBlock2D", "CrossAttnUpBlock2D"),
    block_out_channels=(64, 128, 128), layers_per_block=1,
    attention_head_dim=(1, 2, 2), cross_attention_dim=96, norm_num_groups=32, norm_eps=1e-5,
    flip_sin_to_cos=True, freq_shift=0, transformer_layers_per_block=1,
)

# small SD-1-style config: 8 / 8 / 4 heads of 320 / 640 / 640 channels reach every SD-1.x head dim -- down blocks 40
# and 80, mid block 160, up blocks 80 and 40 (143.7 M parameters)
TINY_SD1_UNET = dict(TINY_UNET, block_out_channels=(320, 640, 640), attention_head_dim=(8, 8, 4))

# tiny SDXL-style config: DownBlock2D first, text_time conditioning, deeper transformer stacks
TINY_XL_UNET = dict(
    sample_size=16, in_channels=4, out_channels=4,
    down_block_types=("DownBlock2D", "CrossAttnDownBlock2D"),
    up_block_types=("CrossAttnUpBlock2D", "UpBlock2D"),
    block_out_channels=(64, 128), layers_per_block=2,
    attention_head_dim=(1, 2), cross_attention_dim=96, norm_num_groups=32, norm_eps=1e-5,
    flip_sin_to_cos=True, freq_shift=0, transformer_layers_per_block=(1, 2),
    addition_embed_type="text_time", addition_time_embed_dim=32,
    projection_class_embeddings_input_dim=64 + 6 * 32,
)

SD21_CONTROLNET = dict(
    in_channels=4, block_out_channels=(320, 640, 1280, 1280), layers_per_block=2,
    down_block_types=("CrossAttnDownBlock2D", "CrossAttnDownBlock2D", "CrossAttnDownBlock2D", "DownBlock2D"),
    attention_head_dim=(5, 10, 20, 20), cross_attention_dim=1024, norm_num_groups=32, norm_eps=1e-5,
    flip_sin_to_cos=True, freq_shift=0, transformer_layers_per_block=1,
    conditioning_embedding_out_channels=(16, 32, 96, 256),
)

# ControlNet for an SD-1.5 base model (lllyasviel/control_v11*_sd15): 8 heads, 768-wide text states
SD15_CONTROLNET = dict(SD21_CONTROLNET, attention_head_dim=8, cross_attention_dim=768)

# SD-1-shaped tiny ControlNet: the down and mid blocks of TINY_SD1_UNET (head dims 40, 80, 160)
TINY_SD1_CONTROLNET = dict(in_channels=4, block_out_channels=(320, 640, 640), layers_per_block=1,
                           down_block_types=("CrossAttnDownBlock2D", "CrossAttnDownBlock2D", "DownBlock2D"),
                           attention_head_dim=(8, 8, 4), cross_attention_dim=96, norm_num_groups=32, norm_eps=1e-5,
                           flip_sin_to_cos=True, freq_shift=0, transformer_layers_per_block=1,
                           conditioning_embedding_out_channels=(16, 32, 96, 256))

TINY_CONTROLNET = dict(
    in_channels=4, block_out_channels=(64, 128, 128), layers_per_block=1,
    down_block_types=("CrossAttnDownBlock2D", "CrossAttnDownBlock2D", "DownBlock2D"),
    attention_head_dim=(1, 2, 2), cross_attention_dim=96, norm_num_groups=32, norm_eps=1e-5,
    flip_sin_to_cos=True, freq_shift=0, transformer_layers_per_block=1,
    conditioning_embedding_out_channels=(16, 32, 96, 256),
)

# ControlNet for SDXL-base (diffusers/controlnet-canny-sdxl-1.0, controlnet-depth-sdxl-1.0): the encoder half of
# SDXL_BASE_UNET with its text_time add-embedding; the mid block takes the last level's depth (10), as diffusers'
# ControlNetModel builds it from transformer_layers_per_block[-1].  9 down residuals + 1 mid residual, the shapes of the
# SDXL UNet's skip connections.
SDXL_CONTROLNET = dict(
    in_channels=4, block_out_channels=(320, 640, 1280), layers_per_block=2,
    down_block_types=("DownBlock2D", "CrossAttnDownBlock2D", "CrossAttnDownBlock2D"),
    attention_head_dim=(5, 10, 20), cross_attention_dim=2048, norm_num_groups=32, norm_eps=1e-5,
    flip_sin_to_cos=True, freq_shift=0, transformer_layers_per_block=(1, 2, 10),
    addition_embed_type="text_time", addition_time_embed_dim=256, projection_class_embeddings_input_dim=2816,
    conditioning_embedding_out_channels=(16, 32, 96, 256),
)

# the encoder half of TINY_XL_UNET (depth-2 mid block)
TINY_XL_CONTROLNET = dict(
    in_channels=4, block_out_channels=(64, 128), layers_per_block=2,
    down_block_types=("DownBlock2D", "CrossAttnDownBlock2D"),
    attention_head_dim=(1, 2), cross_attention_dim=96, norm_num_groups=32, norm_eps=1e-5,
    flip_sin_to_cos=True, freq_shift=0, transformer_layers_per_block=(1, 2),
    addition_embed_type="text_time", addition_time_embed_dim=32, projection_class_embeddings_input_dim=64 + 6 * 32,
    conditioning_embedding_out_channels=(16, 32, 96, 256),
)

SD_VAE = dict(latent_channels=4, out_channels=3, block_out_channels=(128, 256, 512, 512),
              layers_per_block=2, norm_num_groups=32, scaling_factor=0.18215)

# The stock SDXL VAE (SDXL-base 1.0 and the refiner): SD's architecture with other weights; its decoder activations
# exceed fp16's range, so its config sets force_upcast and the pipeline runs it in bf16 (pipeline.vae_dtype).
SDXL_VAE = dict(SD_VAE, scaling_factor=0.13025, force_upcast=True)

TINY_VAE = dict(latent_channels=4, out_channels=3, block_out_channels=(64, 64, 128),
                layers_per_block=1, norm_num_groups=32, scaling_factor=0.18215)


def _as_list(v, n):
    return list(v) if isinstance(v, (list, tuple)) else [v] * n


def _conv(sh, name, co, ci, k, bias=True):
    sh[name + ".weight"] = (co, ci, k, k)
    if bias:
        sh[name + ".bias"] = (co,)


def _norm(sh, name, c):
    sh[name + ".weight"] = (c,)
    sh[name + ".bias"] = (c,)


def _resnet(sh, p, ci, co, temb):
    _norm(sh, p + ".norm1", ci)
    _conv(sh, p + ".conv1", co, ci, 3)
    if temb:
        _conv(sh, p + ".time_emb_proj", co, temb, 1)
    _norm(sh, p + ".norm2", co)
    _conv(sh, p + ".conv2", co, co, 3)
    if ci != co:
        _conv(sh, p + ".conv_shortcut", co, ci, 1)


def _transformer(sh, p, c, ctx_dim, depth):
    _norm(sh, p + ".norm", c)
    _conv(sh, p + ".proj_in", c, c, 1)
    for d in range(depth):
        b = f"{p}.transformer_blocks.{d}"
        for a, kd in (("attn1", c), ("attn2", ctx_dim)):
            _conv(sh, f"{b}.{a}.to_q", c, c, 1, bias=False)
            _conv(sh, f"{b}.{a}.to_k", c, kd, 1, bias=False)
            _conv(sh, f"{b}.{a}.to_v", c, kd, 1, bias=False)
            _conv(sh, f"{b}.{a}.to_out.0", c, c, 1)
        _conv(sh, f"{b}.ff.net.0.proj", 8 * c, c, 1)
        _conv(sh, f"{b}.ff.net.2", c, 4 * c, 1)
        for n in ("norm1", "norm2", "norm3"):
            _norm(sh, f"{b}.{n}", c)
    _conv(sh, p + ".proj_out", c, c, 1)


def unet_param_shapes(cfg) -> "OrderedDict[str, tuple]":
    """name -> shape for every parameter of the reference UNet built from ``cfg``."""
    sh = OrderedDict()
    boc = list(cfg["block_out_channels"])
    nb = len(boc)
    lpb = cfg.get("layers_per_block", 2)
    depth = _as_list(cfg.get("transformer_layers_per_block", 1), nb)
    ctx = cfg["cross_attention_dim"]
    temb = boc[0] * 4
    _conv(sh, "conv_in", boc[0], cfg["in_channels"], 3)
    _conv(sh, "time_embedding.linear_1", temb, boc[0], 1)
    _conv(sh, "time_embedding.linear_2", temb, temb, 1)
    if cfg.get("time_cond_proj_dim"):  # guidance-embedding (LCM) UNets: TimestepEmbedding(cond_proj_dim=...)
        _conv(sh, "time_embedding.cond_proj", boc[0], cfg["time_cond_proj_dim"], 1, bias=False)
    if cfg.get("addition_embed_type") == "text_time":
        _conv(sh, "add_embedding.linear_1", temb, cfg["projection_class_embeddings_input_dim"], 1)
        _conv(sh, "add_embedding.linear_2", temb, temb, 1)
    out = boc[0]
    for i, typ in enumerate(cfg["down_block_types"]):
        inp, out = out, boc[i]
        for j in range(lpb):
            _resnet(sh, f"down_blocks.{i}.resnets.{j}", inp if j == 0 else out, out, temb)
            if typ == "CrossAttnDownBlock2D":
                _transformer(sh, f"down_blocks.{i}.attentions.{j}", out, ctx, depth[i])
        if i != nb - 1:
            _conv(sh, f"down_blocks.{i}.downsamplers.0.conv", out, out, 3)
    _resnet(sh, "mid_block.resnets.0", boc[-1], boc[-1], temb)
    _transformer(sh, "mid_block.attentions.0", boc[-1], ctx, depth[-1])
    _resnet(sh, "mid_block.resnets.1", boc[-1], boc[-1], temb)
    rboc = boc[::-1]
    rdepth = depth[::-1]
    out = rboc[0]
    for i, typ in enumerate(cfg["up_block_types"]):
        prev, out = out, rboc[i]
        inp = rboc[min(i + 1, nb - 1)]
        for j in range(lpb + 1):
            skip = inp if j == lpb else out
            rin = prev if j == 0 else out
            _resnet(sh, f"up_blocks.{i}.resnets.{j}", rin + skip, out, temb)
            if typ == "CrossAttnUpBlock2D":
                _transformer(sh, f"up_blocks.{i}.attentions.{j}", out, ctx, rdepth[i])
        if i != nb - 1:
            _conv(sh, f"up_blocks.{i}.upsamplers.0.conv", out, out, 3)
    _norm(sh, "conv_norm_out", boc[0])
    _conv(sh, "conv_out", cfg["out_channels"], boc[0], 3)
    return sh


def controlnet_param_shapes(cfg) -> "OrderedDict[str, tuple]":
    """name -> shape for the reference ``ControlNetModel`` (controlnet.py:49-189), and for diffusers' ControlNetModel
    where the reference has no counterpart: the ``add_embedding`` of a ``text_time`` (SDXL) config and a mid block of
    depth ``transformer_layers_per_block[-1]`` (1 for every SD 1.x / 2.x ControlNet)."""
    sh = OrderedDict()
    boc = list(cfg["block_out_channels"])
    nb = len(boc)
    lpb = cfg.get("layers_per_block", 2)
    depth = _as_list(cfg.get("transformer_layers_per_block", 1), nb)
    ctx = cfg["cross_attention_dim"]
    temb = boc[0] * 4
    _conv(sh, "conv_in", boc[0], cfg.get("in_channels", 4), 3)
    _conv(sh, "time_embedding.linear_1", temb, boc[0], 1)
    _conv(sh, "time_embedding.linear_2", temb, temb, 1)
    if cfg.get("addition_embed_type") == "text_time":
        _conv(sh, "add_embedding.linear_1", temb, cfg["projection_class_embeddings_input_dim"], 1)
        _conv(sh, "add_embedding.linear_2", temb, temb, 1)
    ce = list(cfg.get("conditioning_embedding_out_channels", (16, 32, 96, 256)))
    _conv(sh, "controlnet_cond_embedding.conv_in", ce[0], 3, 3)
    for i in range(len(ce) - 1):
        _conv(sh, f"controlnet_cond_embedding.blocks.{2 * i}", ce[i], ce[i], 3)
        _conv(sh, f"controlnet_cond_embedding.blocks.{2 * i + 1}", ce[i + 1], ce[i], 3)
    _conv(sh, "controlnet_cond_embedding.conv_out", boc[0], ce[-1], 3)
    k = 0
    _conv(sh, f"controlnet_down_blocks.{k}", boc[0], boc[0], 1)
    out = boc[0]
    for i, typ in enumerate(cfg["down_block_types"]):
        inp, out = out, boc[i]
        for j in range(lpb):
            _resnet(sh, f"down_blocks.{i}.resnets.{j}", inp if j == 0 else out, out, temb)
            if typ == "CrossAttnDownBlock2D":
                _transformer(sh, f"down_blocks.{i}.attentions.{j}", out, ctx, depth[i])
            k += 1
            _conv(sh, f"controlnet_down_blocks.{k}", out, out, 1)
        if i != nb - 1:
            _conv(sh, f"down_blocks.{i}.downsamplers.0.conv", out, out, 3)
            k += 1
            _conv(sh, f"controlnet_down_blocks.{k}", out, out, 1)
    _conv(sh, "controlnet_mid_block", boc[-1], boc[-1], 1)
    _resnet(sh, "mid_block.resnets.0", boc[-1], boc[-1], temb)
    _transformer(sh, "mid_block.attentions.0", boc[-1], ctx, depth[-1])
    _resnet(sh, "mid_block.resnets.1", boc[-1], boc[-1], temb)
    return sh


def check_controlnet_matches_unet(unet_cfg, controlnet_cfg, which="ControlNet"):
    """ValueError naming the first field in which a ControlNet cannot drive the UNet: its residuals must have the
    shapes of the UNet's skip connections (block_out_channels, down_block_types, layers_per_block), it must read the
    same text states (cross_attention_dim) and the same add-embedding inputs (addition_embed_type and, for text_time,
    projection_class_embeddings_input_dim).  Pooled-condition ControlNets (global_pool_conditions) are not
    implemented."""
    if controlnet_cfg.get("global_pool_conditions"):
        raise ValueError(f"{which}: global_pool_conditions=True (pooled residuals) is not supported")
    norm = {"block_out_channels": lambda v: tuple(int(c) for c in v), "down_block_types": lambda v: tuple(v),
            "layers_per_block": int, "cross_attention_dim": int}
    defaults = {"layers_per_block": 2, "addition_embed_type": None}
    fields = ["cross_attention_dim", "block_out_channels", "down_block_types", "layers_per_block", "addition_embed_type"]
    if unet_cfg.get("addition_embed_type") == "text_time":
        fields.append("projection_class_embeddings_input_dim")
    for f in fields:
        u, c = unet_cfg.get(f, defaults.get(f)), controlnet_cfg.get(f, defaults.get(f))
        if f in norm and u is not None and c is not None:
            u, c = norm[f](u), norm[f](c)
        if u != c:
            raise ValueError(f"{which} does not match the UNet: {f} is {c!r}, the UNet's is {u!r}")


def vae_decoder_param_shapes(cfg) -> "OrderedDict[str, tuple]":
    """diffusers ``AutoencoderKL`` decoder + post_quant_conv keys (SURVEY Appendix B1)."""
    sh = OrderedDict()
    boc = list(cfg["block_out_channels"])
    lpb = cfg.get("layers_per_block", 2)
    lc = cfg.get("latent_channels", 4)
    top = boc[-1]
    _conv(sh, "post_quant_conv", lc, lc, 1)
    _conv(sh, "decoder.conv_in", top, lc, 3)
    _resnet(sh, "decoder.mid_block.resnets.0", top, top, 0)
    a = "decoder.mid_block.attentions.0"
    _norm(sh, a + ".group_norm", top)
    for n in ("to_q", "to_k", "to_v", "to_out.0"):
        _conv(sh, f"{a}.{n}", top, top, 1)
    _resnet(sh, "decoder.mid_block.resnets.1", top, top, 0)
    rboc = boc[::-1]
    out = rboc[0]
    for i in range(len(boc)):
        prev, out = out, rboc[i]
        for j in range(lpb + 1):
            _resnet(sh, f"decoder.up_blocks.{i}.resnets.{j}", prev if j == 0 else out, out, 0)
        if i != len(boc) - 1:
            _conv(sh, f"decoder.up_blocks.{i}.upsamplers.0.conv", out, out, 3)
    _norm(sh, "decoder.conv_norm_out", boc[0])
    _conv(sh, "decoder.conv_out", cfg.get("out_channels", 3), boc[0], 3)
    return sh


def vae_encoder_param_shapes(cfg) -> "OrderedDict[str, tuple]":
    """diffusers ``AutoencoderKL`` encoder + quant_conv keys (what ``convert_vae_encoder`` wraps,
    torch2coreml.py:739-749: ``quant_conv(encoder(x))``; double_z: 2 * latent_channels moments)."""
    sh = OrderedDict()
    boc = list(cfg["block_out_channels"])
    lpb = cfg.get("layers_per_block", 2)
    lc = cfg.get("latent_channels", 4)
    _conv(sh, "encoder.conv_in", boc[0], cfg.get("out_channels", 3), 3)
    out = boc[0]
    for i in range(len(boc)):
        prev, out = out, boc[i]
        for j in range(lpb):
            _resnet(sh, f"encoder.down_blocks.{i}.resnets.{j}", prev if j == 0 else out, out, 0)
        if i != len(boc) - 1:
            _conv(sh, f"encoder.down_blocks.{i}.downsamplers.0.conv", out, out, 3)
    top = boc[-1]
    _resnet(sh, "encoder.mid_block.resnets.0", top, top, 0)
    a = "encoder.mid_block.attentions.0"
    _norm(sh, a + ".group_norm", top)
    for n in ("to_q", "to_k", "to_v", "to_out.0"):
        _conv(sh, f"{a}.{n}", top, top, 1)
    _resnet(sh, "encoder.mid_block.resnets.1", top, top, 0)
    _norm(sh, "encoder.conv_norm_out", top)
    _conv(sh, "encoder.conv_out", 2 * lc, top, 3)
    _conv(sh, "quant_conv", 2 * lc, 2 * lc, 1)
    return sh


def random_state_dict(shapes, seed=0, dtype=torch.float32):
    """Deterministic random-init weights with torch's default conv statistics
    (U(-1/sqrt(fan_in), 1/sqrt(fan_in)) for weights and biases) and *non-trivial* norm affines
    (w = 1 + 0.1 n, b = 0.1 n) so that parity tests exercise every term.  There is no network
    for real checkpoints; BASELINE.json asks for random-init weights of the named architecture."""
    g = torch.Generator().manual_seed(seed)
    sd = OrderedDict()
    fan = {}
    for name, shp in shapes.items():
        if len(shp) == 4:
            fan[name.rsplit(".", 1)[0]] = shp[1] * shp[2] * shp[3]
    for name, shp in shapes.items():
        mod = name.rsplit(".", 1)[0]
        if mod in fan:
            b = fan[mod] ** -0.5
            t = (torch.rand(shp, generator=g) * 2 - 1) * b
        elif name.endswith(".weight"):
            t = 1.0 + 0.1 * torch.randn(shp, generator=g)
        else:
            t = 0.1 * torch.randn(shp, generator=g)
        sd[name] = t.to(dtype)
    return sd


# ---------------------------------------------------------------------------------------------------
# CLIP text encoders (transformers.CLIPTextModel, the `text_encoder` the reference converts:
# torch2coreml.py:408-441; called with float input_ids, returns last_hidden_state: pipeline.py:151-175)
# ---------------------------------------------------------------------------------------------------
# SD-2.x: OpenCLIP ViT-H/14 text tower truncated to its penultimate layer (23 layers in the checkpoint's config)
OPENCLIP_H_TEXT = dict(vocab_size=49408, hidden_size=1024, intermediate_size=4096, num_hidden_layers=23,
                       num_attention_heads=16, max_position_embeddings=77, hidden_act="gelu", layer_norm_eps=1e-5)
# SD-1.x: CLIP ViT-L/14 text tower
CLIP_L_TEXT = dict(vocab_size=49408, hidden_size=768, intermediate_size=3072, num_hidden_layers=12,
                   num_attention_heads=12, max_position_embeddings=77, hidden_act="quick_gelu", layer_norm_eps=1e-5)
# SDXL second encoder: OpenCLIP ViT-bigG/14 text tower with text_projection (CLIPTextModelWithProjection)
OPENCLIP_BIGG_TEXT = dict(vocab_size=49408, hidden_size=1280, intermediate_size=5120, num_hidden_layers=32,
                          num_attention_heads=20, max_position_embeddings=77, hidden_act="gelu", layer_norm_eps=1e-5,
                          projection_dim=1280)
TINY_CLIP_TEXT_PROJ = dict(vocab_size=1000, hidden_size=128, intermediate_size=512, num_hidden_layers=3,
                           num_attention_heads=2, max_position_embeddings=77, hidden_act="quick_gelu",
                           layer_norm_eps=1e-5, projection_dim=64)
TINY_CLIP_TEXT = dict(vocab_size=1000, hidden_size=128, intermediate_size=512, num_hidden_layers=2,
                      num_attention_heads=2, max_position_embeddings=77, hidden_act="gelu", layer_norm_eps=1e-5)


def clip_text_param_shapes(cfg):
    """State-dict schema of transformers.CLIPTextModel (names as in the diffusers checkpoints)."""
    d, f = cfg["hidden_size"], cfg["intermediate_size"]
    s = OrderedDict()
    s["text_model.embeddings.token_embedding.weight"] = (cfg["vocab_size"], d)
    s["text_model.embeddings.position_embedding.weight"] = (cfg["max_position_embeddings"], d)
    for i in range(cfg["num_hidden_layers"]):
        p = f"text_model.encoder.layers.{i}."
        for nm in ("q_proj", "k_proj", "v_proj", "out_proj"):
            s[p + f"self_attn.{nm}.weight"] = (d, d)
            s[p + f"self_attn.{nm}.bias"] = (d,)
        for ln in ("layer_norm1", "layer_norm2"):
            s[p + ln + ".weight"] = (d,)
            s[p + ln + ".bias"] = (d,)
        s[p + "mlp.fc1.weight"], s[p + "mlp.fc1.bias"] = (f, d), (f,)
        s[p + "mlp.fc2.weight"], s[p + "mlp.fc2.bias"] = (d, f), (d,)
    s["text_model.final_layer_norm.weight"] = (d,)
    s["text_model.final_layer_norm.bias"] = (d,)
    if cfg.get("projection_dim"):  # CLIPTextModelWithProjection
        s["text_projection.weight"] = (cfg["projection_dim"], d)
    return s


def random_clip_text_state_dict(cfg, seed=0, dtype=torch.float32):
    """Random-init text-encoder weights: U(+-1/sqrt(fan_in)) linears, N(0, 1) embeddings scaled to unit-ish
    activations, non-trivial LayerNorm affines (same conventions as random_state_dict)."""
    g = torch.Generator().manual_seed(seed)
    sd = OrderedDict()
    for name, shp in clip_text_param_shapes(cfg).items():
        if "embedding" in name:
            t = 0.5 * torch.randn(shp, generator=g)
        elif "layer_norm" in name:
            t = (1.0 + 0.1 * torch.randn(shp, generator=g)) if name.endswith("weight") else 0.1 * torch.randn(shp, generator=g)
        elif len(shp) == 2:
            t = (torch.rand(shp, generator=g) * 2 - 1) * shp[1] ** -0.5
        else:
            t = 0.1 * torch.randn(shp, generator=g)
        sd[name] = t.to(dtype)
    return sd


# ---------------------------------------------------------------------------------------------------
# Stable Diffusion safety checker (diffusers' StableDiffusionSafetyChecker: a transformers.CLIPVisionModel, a bias-free
# visual projection and 17 + 3 concept embeddings with thresholds; the reference converts it with forward_coreml,
# torch2coreml.py:1177-1209, and runs it after the VAE decode, pipeline.py:286-311)
# ---------------------------------------------------------------------------------------------------
# transformers.CLIPVisionConfig() defaults: they fill the keys a checkpoint's `vision_config` leaves out
CLIP_VISION_DEFAULTS = dict(hidden_size=768, intermediate_size=3072, num_hidden_layers=12, num_attention_heads=12,
                            num_channels=3, image_size=224, patch_size=32, hidden_act="quick_gelu", layer_norm_eps=1e-5)
# CLIPConfig's default projection_dim (the checkpoint's top-level "projection_dim" overrides it)
CLIP_PROJECTION_DIM_DEFAULT = 512
# CompVis/stable-diffusion-safety-checker, shipped as `safety_checker/` with SD 1.4 / 1.5: ViT-L/14 at 224
SD_SAFETY_CHECKER = dict(CLIP_VISION_DEFAULTS, hidden_size=1024, intermediate_size=4096, num_hidden_layers=24,
                         num_attention_heads=16, patch_size=14, projection_dim=768, num_concepts=17,
                         num_special_concepts=3)
TINY_SAFETY_CHECKER = dict(CLIP_VISION_DEFAULTS, hidden_size=128, intermediate_size=512, num_hidden_layers=2,
                           num_attention_heads=2, patch_size=14, projection_dim=64, num_concepts=17,
                           num_special_concepts=3)


def safety_checker_config(raw: dict) -> dict:
    """A ``safety_checker/config.json`` (a CLIPConfig) -> the flat config the engine reads: the ``vision_config`` keys
    over CLIP_VISION_DEFAULTS, the top-level ``projection_dim``, and StableDiffusionSafetyChecker's fixed 17 + 3
    concept rows."""
    vis = raw.get("vision_config") or {}
    cfg = dict(CLIP_VISION_DEFAULTS)
    cfg.update({k: vis[k] for k in CLIP_VISION_DEFAULTS if k in vis})
    cfg["projection_dim"] = raw.get("projection_dim", CLIP_PROJECTION_DIM_DEFAULT)
    cfg["num_concepts"], cfg["num_special_concepts"] = 17, 3
    return cfg


def safety_checker_param_shapes(cfg):
    """State-dict schema of StableDiffusionSafetyChecker (its CLIPVisionModel sits under ``vision_model.``)."""
    d, f, p, c = cfg["hidden_size"], cfg["intermediate_size"], cfg["patch_size"], cfg["num_channels"]
    g = cfg["image_size"] // p
    proj = cfg["projection_dim"]
    v = "vision_model.vision_model."
    s = OrderedDict()
    s[v + "embeddings.class_embedding"] = (d,)
    s[v + "embeddings.patch_embedding.weight"] = (d, c, p, p)
    s[v + "embeddings.position_embedding.weight"] = (g * g + 1, d)
    s[v + "pre_layrnorm.weight"], s[v + "pre_layrnorm.bias"] = (d,), (d,)
    for i in range(cfg["num_hidden_layers"]):
        q = f"{v}encoder.layers.{i}."
        for nm in ("q_proj", "k_proj", "v_proj", "out_proj"):
            s[q + f"self_attn.{nm}.weight"] = (d, d)
            s[q + f"self_attn.{nm}.bias"] = (d,)
        for ln in ("layer_norm1", "layer_norm2"):
            s[q + ln + ".weight"] = (d,)
            s[q + ln + ".bias"] = (d,)
        s[q + "mlp.fc1.weight"], s[q + "mlp.fc1.bias"] = (f, d), (f,)
        s[q + "mlp.fc2.weight"], s[q + "mlp.fc2.bias"] = (d, f), (d,)
    s[v + "post_layernorm.weight"], s[v + "post_layernorm.bias"] = (d,), (d,)
    s["visual_projection.weight"] = (proj, d)
    s["concept_embeds"] = (cfg["num_concepts"], proj)
    s["special_care_embeds"] = (cfg["num_special_concepts"], proj)
    s["concept_embeds_weights"] = (cfg["num_concepts"],)
    s["special_care_embeds_weights"] = (cfg["num_special_concepts"],)
    return s


SAFETY_CONCEPT_KEYS = ("concept_embeds", "special_care_embeds", "concept_embeds_weights", "special_care_embeds_weights")


def random_safety_checker_state_dict(cfg, seed=0, dtype=torch.float32):
    """Random-init safety-checker weights (conventions of random_clip_text_state_dict; the patch embedding is a conv,
    U(+-1/sqrt(fan_in))).  The concept tables are fp32 whatever ``dtype`` is: N(0, 1) embeddings and thresholds of
    4 to 5 / sqrt(projection_dim), four standard deviations or more above the cosine of a random direction with them,
    so random images are not flagged."""
    g = torch.Generator().manual_seed(seed)
    sd = OrderedDict()
    for name, shp in safety_checker_param_shapes(cfg).items():
        if name in SAFETY_CONCEPT_KEYS:
            t = torch.randn(shp, generator=g) if len(shp) == 2 else \
                (4 + torch.rand(shp, generator=g)) * cfg["projection_dim"] ** -0.5
            sd[name] = t.float()
            continue
        if "embedding" in name and len(shp) != 4:
            t = 0.5 * torch.randn(shp, generator=g)
        elif any(k in name for k in ("layer_norm", "layrnorm", "layernorm")):
            t = (1.0 + 0.1 * torch.randn(shp, generator=g)) if name.endswith("weight") else 0.1 * torch.randn(shp, generator=g)
        elif len(shp) == 4:
            t = (torch.rand(shp, generator=g) * 2 - 1) * (shp[1] * shp[2] * shp[3]) ** -0.5
        elif len(shp) == 2:
            t = (torch.rand(shp, generator=g) * 2 - 1) * shp[1] ** -0.5
        else:
            t = 0.1 * torch.randn(shp, generator=g)
        sd[name] = t.to(dtype)
    return sd
