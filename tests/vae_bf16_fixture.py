"""Homogeneous-scaling fixture for the bf16 VAE: random VAE decoder weights rescaled so that the decoder's residual
stream is S = 2^k times larger while the image stays the same.

conv_in, every ResNet conv2 and the mid attention's to_out.0 are multiplied (weight and bias) by S; conv_shortcut and
the upsampler convolutions only get their bias multiplied, since their input already carries S.  GroupNorm is scale
invariant (up to its eps), so every normalised branch sees the unscaled values, every branch added to the stream
comes out S times larger, and conv_norm_out removes S again before conv_out.  k is chosen from the oracle's stream
maximum so that the scaled stream reaches >= 4 x 65504: far past fp16's range, well inside bf16's."""
import math

import torch

FP16_MAX = 65504.0
TARGET = 4 * FP16_MAX


def scaled_state_dict(sd, k):
    s = float(2 ** k)
    out = dict(sd)
    for key, v in sd.items():
        if not key.startswith("decoder."):
            continue
        full = (key.startswith("decoder.conv_in.") or ".conv2." in key or
                (".attentions." in key and ".to_out.0." in key))
        bias_only = (".conv_shortcut." in key or ".upsamplers." in key) and key.endswith(".bias")
        if full or bias_only:
            out[key] = (v.float() * s).to(v.dtype)
    return out


def stream_max(R, sd, cfg, z):
    """max |residual stream| of the oracle decoder (outputs of conv_in, every ResNet, the attention and the
    upsampler convolutions) and the image."""
    seen = []
    res0, attn0, conv0 = R._vae_resnet, R._vae_attn, R._conv

    def resnet(sd_, p, x):
        y = res0(sd_, p, x)
        seen.append(float(y.abs().max()))
        return y

    def attn(sd_, p, x):
        y = attn0(sd_, p, x)
        seen.append(float(y.abs().max()))
        return y

    def conv(sd_, p, x, *a, **kw):
        y = conv0(sd_, p, x, *a, **kw)
        if p == "decoder.conv_in" or ".upsamplers." in p:
            seen.append(float(y.abs().max()))
        return y

    R._vae_resnet, R._vae_attn, R._conv = resnet, attn, conv
    try:
        with torch.no_grad():
            img = R.vae_decode(sd, cfg, z)
    finally:
        R._vae_resnet, R._vae_attn, R._conv = res0, attn0, conv0
    return max(seen), img


def pick_k(stream):
    """Smallest k with 2^k * stream >= TARGET."""
    return max(1, math.ceil(math.log2(TARGET / stream)))
