"""CPU oracle of the Stable Diffusion safety checker.  Test infrastructure only.

* :func:`library_forward`: ``transformers.CLIPVisionModel`` (eager attention, fp32) + the visual projection -- the
  network diffusers' ``StableDiffusionSafetyChecker`` wraps;
* :func:`clip_vision_forward`: a plain restatement of it, pinned to the library in ``tests/test_safety_checker.py``;
* :func:`head`: the ``forward_coreml`` head the reference converts (``torch2coreml.py:1177-1209``), in float64 by default;
* :func:`preprocess`: ``feature_extractor(numpy_to_pil(image))`` of transformers 4.44.2 -- Pillow's BICUBIC resize
  of the shortest edge, centre crop, then rescale ``float32(float64(u8) * (1/255))`` and ``(v - mean) / std`` in
  float32, in numpy (the installed transformers release computes a slightly different resize);
* :func:`resample_u8`: an integer resampler that applies fixed-point coefficient tables the way Pillow does, so that
  the host tables can be pinned to ``PIL.Image.resize`` without a GPU.
"""
from __future__ import annotations

import math

import numpy as np
import torch
import torch.nn.functional as F

V = "vision_model.vision_model."


def build_library_model(cfg, sd):
    from transformers import CLIPVisionConfig, CLIPVisionModel

    conf = CLIPVisionConfig(hidden_size=cfg["hidden_size"], intermediate_size=cfg["intermediate_size"],
                            num_hidden_layers=cfg["num_hidden_layers"], num_attention_heads=cfg["num_attention_heads"],
                            num_channels=cfg["num_channels"], image_size=cfg["image_size"],
                            patch_size=cfg["patch_size"], hidden_act=cfg["hidden_act"],
                            layer_norm_eps=cfg["layer_norm_eps"])
    conf._attn_implementation = "eager"
    model = CLIPVisionModel(conf).eval()
    vsd = {k[len("vision_model."):]: v.float() for k, v in sd.items() if k.startswith(V)}
    missing, unexpected = model.load_state_dict(vsd, strict=False)
    bad = [k for k in missing if "position_ids" not in k]
    if bad or unexpected:
        raise RuntimeError(f"state dict mismatch: missing {bad} unexpected {unexpected}")
    return model


def library_forward(cfg, sd, pixel_values):
    """-> dict(last_hidden_state [B, T, D], pooler_output [B, D], image_embeds [B, P]), fp32."""
    model = build_library_model(cfg, sd)
    with torch.no_grad():
        o = model(pixel_values=pixel_values.float())
        emb = F.linear(o.pooler_output, sd["visual_projection.weight"].float())
    return {"last_hidden_state": o.last_hidden_state, "pooler_output": o.pooler_output, "image_embeds": emb}


def clip_vision_forward(cfg, sd, pixel_values, dtype=torch.float32):
    """Restatement of transformers' CLIPVisionTransformer + the visual projection: conv patch embedding, class token,
    position embeddings, pre_layrnorm, pre-LN blocks with full self-attention, post_layernorm of the class token."""
    d, heads, eps, p = cfg["hidden_size"], cfg["num_attention_heads"], cfg["layer_norm_eps"], cfg["patch_size"]
    f = {k: v.to(dtype) for k, v in sd.items()}
    x = pixel_values.to(dtype)
    b = x.shape[0]
    pe = F.conv2d(x, f[V + "embeddings.patch_embedding.weight"], stride=p).flatten(2).transpose(1, 2)
    cls = f[V + "embeddings.class_embedding"].expand(b, 1, d)
    x = torch.cat([cls, pe], 1) + f[V + "embeddings.position_embedding.weight"]
    s = x.shape[1]
    x = F.layer_norm(x, (d,), f[V + "pre_layrnorm.weight"], f[V + "pre_layrnorm.bias"], eps)
    act = (lambda t: t * torch.sigmoid(1.702 * t)) if cfg["hidden_act"] == "quick_gelu" else F.gelu
    for i in range(cfg["num_hidden_layers"]):
        q_ = f"{V}encoder.layers.{i}."
        h = F.layer_norm(x, (d,), f[q_ + "layer_norm1.weight"], f[q_ + "layer_norm1.bias"], eps)
        q, k, v = (F.linear(h, f[q_ + f"self_attn.{n}.weight"], f[q_ + f"self_attn.{n}.bias"])
                   .view(b, s, heads, d // heads).transpose(1, 2) for n in ("q_proj", "k_proj", "v_proj"))
        att = torch.softmax(q @ k.transpose(-1, -2) / math.sqrt(d // heads), dim=-1) @ v
        x = x + F.linear(att.transpose(1, 2).reshape(b, s, d), f[q_ + "self_attn.out_proj.weight"],
                         f[q_ + "self_attn.out_proj.bias"])
        h = F.layer_norm(x, (d,), f[q_ + "layer_norm2.weight"], f[q_ + "layer_norm2.bias"], eps)
        x = x + F.linear(act(F.linear(h, f[q_ + "mlp.fc1.weight"], f[q_ + "mlp.fc1.bias"])), f[q_ + "mlp.fc2.weight"],
                         f[q_ + "mlp.fc2.bias"])
    pooled = F.layer_norm(x[:, 0], (d,), f[V + "post_layernorm.weight"], f[V + "post_layernorm.bias"], eps)
    return {"last_hidden_state": x, "pooler_output": pooled,
            "image_embeds": F.linear(pooled, f["visual_projection.weight"])}


def head(image_embeds, sd, adjustment=0.0, dtype=torch.float64):
    """forward_coreml's head (torch2coreml.py:1181-1203): -> (concept_scores [B, 17], has_nsfw bool [B]).  No 3-decimal
    rounding: that is in diffusers' eager forward, not in the graph the reference runs."""
    def cos(a, b):
        return F.normalize(a.to(dtype)) @ F.normalize(b.to(dtype)).t()

    special = cos(image_embeds, sd["special_care_embeds"]) - sd["special_care_embeds_weights"].to(dtype) + adjustment
    care = special.gt(0).float().sum(1).gt(0).to(dtype)
    scores = cos(image_embeds, sd["concept_embeds"]) - sd["concept_embeds_weights"].to(dtype) + (care * 0.01)[:, None]
    return scores, scores.gt(0).any(1)


def preprocess(images_u8, size=224, crop=(224, 224), mean=(0.48145466, 0.4578275, 0.40821073),
               std=(0.26862954, 0.26130258, 0.27577711)):
    """u8 NHWC [B, H, W, 3] -> fp32 pixel_values [B, 3, crop_h, crop_w] exactly as CLIPImageProcessor 4.44.2 computes
    them from PIL images."""
    from PIL import Image

    out = []
    for im in np.asarray(images_u8):
        h, w = im.shape[:2]
        short, long = (w, h) if w <= h else (h, w)
        new_long = int(size * long / short)
        nh, nw = (new_long, size) if w <= h else (size, new_long)
        r = np.asarray(Image.fromarray(im).resize((nw, nh), resample=Image.BICUBIC))
        top, left = (nh - crop[0]) // 2, (nw - crop[1]) // 2
        r = r[top:top + crop[0], left:left + crop[1]]
        v = (r.astype(np.float64) * (1 / 255)).astype(np.float32)
        v = (v - np.array(mean, dtype=np.float32)) / np.array(std, dtype=np.float32)
        out.append(v.transpose(2, 0, 1))
    return np.stack(out).astype(np.float32)


def resample_u8(img, h_table, v_table):
    """Applies (bounds, coeffs) fixed-point tables to a u8 [H, W, C] image: horizontal pass, u8 intermediate, then the
    vertical pass; accumulators start at 2^21 and are shifted right by 22 and saturated."""
    def apply(x, bounds, coeffs):  # resample axis 1 of x [A, N, C]
        out = np.empty((x.shape[0], len(bounds), x.shape[2]), np.uint8)
        for i, (lo, n) in enumerate(bounds):
            acc = (x[:, lo:lo + n].astype(np.int64) * coeffs[i, :n].astype(np.int64)[None, :, None]).sum(1) + (1 << 21)
            out[:, i] = np.clip(acc >> 22, 0, 255)
        return out
    tmp = apply(np.asarray(img), *h_table)
    return apply(tmp.transpose(1, 0, 2), *v_table).transpose(1, 0, 2)
