"""Restatement of an SDXL (``text_time``) ControlNet forward in fp32, composed of the blocks of ``oracle.restated``.

The reference ControlNetModel (controlnet.py:199-250) has no SDXL variant; diffusers' ControlNetModel differs from it in
two places, both restated here:
* the time embedding gains the add-embedding of ``time_ids`` / ``text_embeds``, computed as
  ``UNet2DConditionModelXL.forward`` computes it (unet.py:1072-1084);
* the mid block's transformer has depth ``transformer_layers_per_block[-1]`` (10 for SDXL).
Everything else is ``restated.controlnet_forward``'s sequence.  tests/test_controlnet_xl.py pins this restatement to
the fixtures of the unmodified reference modules (tests/golden/make_golden_controlnet_xl.py)."""
import torch
import torch.nn.functional as F

from oracle import restated as R


def controlnet_forward_xl(sd, cfg, sample, timestep, encoder_hidden_states, controlnet_cond, time_ids, text_embeds):
    """-> the list of down residuals followed by the mid residual (fp32, or fp64 given fp64 weights and inputs)."""
    boc = list(cfg["block_out_channels"])
    nb = len(boc)
    lpb = cfg.get("layers_per_block", 2)
    heads = R._as_list(cfg.get("attention_head_dim", 8), nb)
    depth = R._as_list(cfg.get("transformer_layers_per_block", 1), nb)
    groups = cfg.get("norm_num_groups", 32)
    eps = cfg.get("norm_eps", 1e-5)
    flip, shift = cfg.get("flip_sin_to_cos", True), cfg.get("freq_shift", 0)
    ctx = R._f(encoder_hidden_states)
    temb = R._time_mlp(sd, "time_embedding", R.timestep_embedding(timestep, boc[0], flip, shift))
    te = R.timestep_embedding(time_ids.flatten(), cfg["addition_time_embed_dim"], flip, shift)
    te = te.reshape(text_embeds.shape[0], -1)
    temb = temb + R._time_mlp(sd, "add_embedding", torch.cat([R._f(text_embeds), te], dim=-1))
    ce = list(cfg.get("conditioning_embedding_out_channels", (16, 32, 96, 256)))
    e = F.silu(R._conv(sd, "controlnet_cond_embedding.conv_in", R._f(controlnet_cond), padding=1))
    for i in range(len(ce) - 1):
        e = F.silu(R._conv(sd, f"controlnet_cond_embedding.blocks.{2 * i}", e, padding=1))
        e = F.silu(R._conv(sd, f"controlnet_cond_embedding.blocks.{2 * i + 1}", e, stride=2, padding=1))
    e = R._conv(sd, "controlnet_cond_embedding.conv_out", e, padding=1)
    x = R._conv(sd, "conv_in", R._f(sample), padding=1) + e
    skips = [x]
    for i, typ in enumerate(cfg["down_block_types"]):
        for j in range(lpb):
            x = R._resnet(sd, f"down_blocks.{i}.resnets.{j}", x, temb, groups, eps)
            if typ == "CrossAttnDownBlock2D":
                x = R._spatial_transformer(sd, f"down_blocks.{i}.attentions.{j}", x, ctx, heads[i], depth[i])
            skips.append(x)
        if i != nb - 1:
            x = R._conv(sd, f"down_blocks.{i}.downsamplers.0.conv", x, stride=2, padding=1)
            skips.append(x)
    x = R._resnet(sd, "mid_block.resnets.0", x, temb, groups, eps)
    x = R._spatial_transformer(sd, "mid_block.attentions.0", x, ctx, heads[-1], depth[-1])
    x = R._resnet(sd, "mid_block.resnets.1", x, temb, groups, eps)
    outs = [R._conv(sd, f"controlnet_down_blocks.{k}", s) for k, s in enumerate(skips)]
    outs.append(R._conv(sd, "controlnet_mid_block", x))
    return outs
