"""Fake-quant oracle of the W8A8 UNet: oracle.restated.unet_forward with the recipe's convolutions replaced by their
int8 form in float64 (quantized activations and weights, exact integer products, scales applied after the sum)."""
import contextlib

import torch
import torch.nn.functional as F

from oracle import restated as R


def qconv(x, w, b, s_a, padding=1):
    """The W8A8 convolution in float64: clamp(rne(x / s_a)) (*) clamp(rne(W / s_w)) * s_a * s_w + b.  Integer products
    of |q| <= 127 summed over K <= 23040 terms stay below 2^53, so the float64 sum is the exact integer sum."""
    x, w = x.double(), w.double()
    s_w = w.reshape(w.shape[0], -1).abs().amax(1) / 127
    s_w = torch.where(s_w > 0, s_w, torch.ones_like(s_w))
    qa = torch.clamp(torch.round(x / s_a), -127, 127)
    qw = torch.clamp(torch.round(w / s_w[:, None, None, None]), -127, 127)
    acc = F.conv2d(qa, qw, None, padding=padding)
    out = acc * (s_a * s_w)[None, :, None, None]
    return out if b is None else out + b.double()[None, :, None, None]


@contextlib.contextmanager
def quantized(scales):
    """Within the block, restated._conv runs the layers of `scales` (name -> s_a) as W8A8."""
    orig = R._conv

    def conv(sd, prefix, x, stride=1, padding=0):
        if prefix in scales:
            return qconv(x, R._w(sd, prefix + ".weight"), sd.get(prefix + ".bias"), scales[prefix], padding).to(x.dtype)
        return orig(sd, prefix, x, stride=stride, padding=padding)

    R._conv = conv
    try:
        yield
    finally:
        R._conv = orig


def unet_forward_q(sd, cfg, sample, timestep, ctx, scales, **kw):
    with quantized(scales):
        return R.unet_forward(sd, cfg, sample, timestep, ctx, **kw)


def calibrate(sd, cfg, sample, timestep, ctx, layers, **kw):
    """max |x| at the input of each of `layers` in one oracle forward."""
    amax = {}
    orig = R._conv

    def conv(sd_, prefix, x, stride=1, padding=0):
        if prefix in layers:
            amax[prefix] = max(amax.get(prefix, 0.0), float(x.abs().max()))
        return orig(sd_, prefix, x, stride=stride, padding=padding)

    R._conv = conv
    try:
        R.unet_forward(sd, cfg, sample, timestep, ctx, **kw)
    finally:
        R._conv = orig
    return amax
