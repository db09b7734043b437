"""Golden fixtures of the SDXL ControlNet (config.SDXL_CONTROLNET, diffusers/controlnet-canny-sdxl-1.0's shape) and of
its tiny counterpart (config.TINY_XL_CONTROLNET), produced on the CPU in fp32 by UNMODIFIED reference modules
(python_coreml_stable_diffusion.{controlnet,unet}, imported through oracle/ref_unet.py).  The reference ControlNetModel
has no SDXL variant, so the network is composed of its parts the way diffusers' ControlNetModel builds it:

  * the reference ControlNetModel: conditioning embedder, conv_in, time embedding, down blocks and zero convolutions;
  * a reference UNetMidBlock2DCrossAttn(transformer_layers_per_block=depth[-1]) as its mid block (the reference
    ControlNetModel builds a depth-1 mid block);
  * reference Timesteps + TimestepEmbedding as add_time_proj / add_embedding, added to the time embedding the way
    UNet2DConditionModelXL.forward adds them.

Run where the reference tree is present:

    python tests/golden/make_golden_controlnet_xl.py

Weights are regenerated from the seed on the test side (see make_golden.py); each fixture stores the seeds, a weight
fingerprint and the sha256 of the composed module's parameter schema.  controlnet_tiny_xl.npz keeps the fp32
residuals whole; controlnet_sdxl.npz (32x32 latents, a 256x256 condition image, fp16 weights) keeps them at fp16,
sub-sampled [:, :, ::STRIDE, ::STRIDE] like controlnet_sd21.npz.
"""
import hashlib
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

from b200sd import config  # noqa: E402
from oracle import ref_unet  # noqa: E402
from make_golden import fingerprint  # noqa: E402

OUT = os.path.dirname(os.path.abspath(__file__))
STRIDE = 4  # controlnet_sdxl.npz: residuals sub-sampled [:, :, ::STRIDE, ::STRIDE]
TIMESTEP = 501.0


def schema_digest(shapes):
    lines = "\n".join(f"{k} {tuple(int(d) for d in v)}" for k, v in sorted(shapes.items()))
    return hashlib.sha256(lines.encode()).hexdigest()


class _TimeEmbeddingWithAdd(torch.nn.Module):
    """The ControlNet's own time_embedding followed by ``+ add_embedding(cat(text_embeds, add_time_proj(time_ids)))``,
    as UNet2DConditionModelXL.forward (unet.py:1072-1084) computes emb; the inputs are set per call."""

    def __init__(self, time_embedding, add_time_proj, add_embedding):
        super().__init__()
        self.time_embedding, self.add_time_proj, self.add_embedding = time_embedding, add_time_proj, add_embedding
        self.time_ids = self.text_embeds = None

    def forward(self, t_emb):
        emb = self.time_embedding(t_emb)
        time_embeds = self.add_time_proj(self.time_ids.flatten()).reshape((self.text_embeds.shape[0], -1))
        return emb + self.add_embedding(torch.concat([self.text_embeds, time_embeds], dim=-1))


def build(cfg, meta=False):
    """The composed SDXL ControlNet (parameters under diffusers' names)."""
    ref = ref_unet.load()
    boc = list(cfg["block_out_channels"])
    nb = len(boc)
    depth = config._as_list(cfg["transformer_layers_per_block"], nb)
    heads = config._as_list(cfg["attention_head_dim"], nb)
    temb = boc[0] * 4
    with torch.device("meta" if meta else "cpu"):
        cn = ref.controlnet.ControlNetModel(**cfg).eval()
        cn.mid_block = ref.unet.UNetMidBlock2DCrossAttn(
            in_channels=boc[-1], temb_channels=temb, resnet_eps=cfg["norm_eps"], resnet_act_fn="silu",
            output_scale_factor=1, resnet_time_scale_shift="default", cross_attention_dim=cfg["cross_attention_dim"],
            attn_num_head_channels=heads[-1], resnet_groups=cfg["norm_num_groups"],
            transformer_layers_per_block=depth[-1]).eval()
        cn.add_time_proj = ref.unet.Timesteps(cfg["addition_time_embed_dim"], cfg["flip_sin_to_cos"], cfg["freq_shift"])
        cn.add_embedding = ref.unet.TimestepEmbedding(cfg["projection_class_embeddings_input_dim"], temb).eval()
    return cn


def run(cn, x, t, ctx, cond, time_ids, text_embeds):
    """The reference ControlNetModel.forward with the add-embedding in its time embedding."""
    plain = cn.time_embedding
    wrapped = _TimeEmbeddingWithAdd(plain, cn.add_time_proj, cn.add_embedding)
    wrapped.time_ids, wrapped.text_embeds = time_ids, text_embeds
    cn.time_embedding = wrapped
    try:
        with torch.no_grad():
            down, mid = cn(x, t, ctx, cond)
    finally:
        cn.time_embedding = plain
    return list(down) + [mid]


def inputs(cfg, seed, size, pooled):
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(2, cfg["in_channels"], size, size, generator=g)
    ctx = torch.randn(2, cfg["cross_attention_dim"], 1, 77, generator=g)
    text_embeds = torch.randn(2, pooled, generator=g)
    time_ids = torch.tensor([[8.0 * size, 8.0 * size, 0.0, 0.0, 8.0 * size, 8.0 * size],
                             [8.0 * size, 4.0 * size, 16.0, 8.0, 8.0 * size, 8.0 * size]])
    return x, ctx, text_embeds, time_ids


def make(name, cfg, wseed, iseed, cseed, size, fp16, stride):
    pooled = cfg["projection_class_embeddings_input_dim"] - 6 * cfg["addition_time_embed_dim"]
    shapes = config.controlnet_param_shapes(cfg)
    sd = config.random_state_dict(shapes, seed=wseed, dtype=torch.float16 if fp16 else torch.float32)
    digest = schema_digest({k: v.shape for k, v in build(cfg, meta=True).state_dict().items()})
    assert digest == schema_digest(shapes), f"{name}: config.controlnet_param_shapes differs from the reference modules"
    cn = build(cfg)
    cn.load_state_dict({k: v.clone().float() for k, v in sd.items()})
    x, ctx, text_embeds, time_ids = inputs(cfg, iseed, size, pooled)
    cond = torch.rand(2, 3, 8 * size, 8 * size, generator=torch.Generator().manual_seed(cseed))
    if fp16:
        x, ctx, text_embeds, cond = (v.half().float() for v in (x, ctx, text_embeds, cond))
    res = run(cn, x, torch.tensor([TIMESTEP, TIMESTEP]), ctx, cond, time_ids, text_embeds)
    print(name, [tuple(r.shape) for r in res], [round(float(r.abs().max()), 3) for r in res])
    dt = np.float16 if fp16 else np.float32
    np.savez_compressed(os.path.join(OUT, f"{name}.npz"), weight_seed=wseed, input_seed=iseed, cond_seed=cseed,
                        size=size, stride=stride, timestep=TIMESTEP, fingerprint=fingerprint(sd),
                        schema=np.array(digest), time_ids=time_ids.numpy(),
                        **{f"residual_{i}": r[:, :, ::stride, ::stride].numpy().astype(dt) for i, r in enumerate(res)})


def main():
    assert ref_unet.available(), "reference tree not importable"
    make("controlnet_tiny_xl", config.TINY_XL_CONTROLNET, 61, 62, 63, 16, fp16=False, stride=1)
    make("controlnet_sdxl", config.SDXL_CONTROLNET, 71, 72, 73, 32, fp16=True, stride=STRIDE)


if __name__ == "__main__":
    main()
