"""W8A8 quantization of the UNet's ResNet and up-sampler 3x3 convolutions (int8 weights and activations on the int8
wgmma kernel, ``lib.conv3x3_s8``).

Semantics (restated from the reference's ``activation_quantization.py``; not bit-parity with coremltools):
  * weights: symmetric int8 per output channel, s_w[n] = max_k |W[n, k]| / 127 (an all-zero row gets scale 1),
    q = clamp(rne(W / s_w), -127, 127);
  * activations: symmetric int8 per tensor, s_a = amax / 127, where amax is max |x| at the layer's input over every UNet
    call of a calibration run with the fp16 engine (``B200StableDiffusionPipeline.calibrate_unet``).  For a ResNet
    convolution x is the GroupNorm + SiLU output, for an up-sampler convolution the tensor before the upsample;
  * epilogue: out = fp16(float(acc_i32) * (s_a * s_w[n]) + bias + residual).
Only layers named in a recipe are quantized; every other layer stays the fp16 launch it would be without a recipe.
(The reference keeps skipped layers as int8-weight / float-activation layers; here they stay fp16.)
"""
from __future__ import annotations

import json
import math
import re

import torch

# the reference's sensitivity JSON (README "Activation Quantization", step 2) and the module names it uses
_ELIGIBLE = re.compile(r"^(down_blocks\.\d+\.resnets\.\d+\.conv[12]|mid_block\.resnets\.\d+\.conv[12]|"
                       r"up_blocks\.\d+\.resnets\.\d+\.conv[12]|up_blocks\.\d+\.upsamplers\.0\.conv)$")
_ARCH_KEYS = ("block_out_channels", "layers_per_block", "down_block_types", "up_block_types", "in_channels")


def architecture(cfg: dict) -> dict:
    """The parts of a UNet config a recipe's layer names and scales depend on."""
    out = {}
    for k in _ARCH_KEYS:
        v = cfg.get(k)
        out[k] = list(v) if isinstance(v, (list, tuple)) else v
    out["layers_per_block"] = cfg.get("layers_per_block", 2)
    out["in_channels"] = cfg.get("in_channels", 4)
    return out


def quantizable_layers(cfg: dict) -> "dict[str, int]":
    """Every layer this engine can run in W8A8 for a UNet config -> its input channel count, in launch order."""
    boc = list(cfg["block_out_channels"])
    nb, lpb = len(boc), cfg.get("layers_per_block", 2)
    out = {}
    ch = boc[0]
    skip_ch = [ch]
    for i in range(nb):
        for j in range(lpb):
            out[f"down_blocks.{i}.resnets.{j}.conv1"] = ch
            out[f"down_blocks.{i}.resnets.{j}.conv2"] = boc[i]
            ch = boc[i]
            skip_ch.append(ch)
        if i != nb - 1:
            skip_ch.append(ch)
    for j in range(2):
        out[f"mid_block.resnets.{j}.conv1"] = ch
        out[f"mid_block.resnets.{j}.conv2"] = ch
    rboc = boc[::-1]
    for i in range(nb):
        for j in range(lpb + 1):
            out[f"up_blocks.{i}.resnets.{j}.conv1"] = ch + skip_ch.pop()
            out[f"up_blocks.{i}.resnets.{j}.conv2"] = rboc[i]
            ch = rboc[i]
        if i != nb - 1:
            out[f"up_blocks.{i}.upsamplers.0.conv"] = ch
    return out


def quantize_weight(w: torch.Tensor):
    """Symmetric per-output-channel int8 of a [Cout, ...] weight: (q int8 [Cout, ...], s_w fp32 [Cout]).
    s_w[n] = max |W[n]| / 127 (1 for an all-zero row); q = clamp(round-half-even(W / s_w), -127, 127)."""
    wf = w.detach().to(torch.float32)
    flat = wf.reshape(wf.shape[0], -1)
    amax = flat.abs().amax(dim=1)
    s = torch.where(amax > 0, amax / 127.0, torch.ones_like(amax))
    q = torch.clamp(torch.round(flat / s[:, None]), -127, 127).to(torch.int8)  # torch.round: half to even
    return q.reshape(wf.shape), s


def quantize_activation(x: torch.Tensor, scale: float) -> torch.Tensor:
    """Symmetric per-tensor int8 of activations with s_a = scale: clamp(round-half-even(x / s_a), -127, 127)."""
    return torch.clamp(torch.round(x / scale), -127, 127)


class W8A8Recipe:
    """Layer name -> activation scale s_a (amax / 127) of every layer to run in W8A8, plus the architecture the scales
    were calibrated on."""

    def __init__(self, scales: "dict[str, float]", arch: "dict | None" = None):
        self.scales = {str(k): float(v) for k, v in scales.items()}
        self.arch = arch

    @classmethod
    def from_amax(cls, amax: "dict[str, float]", cfg: dict) -> "W8A8Recipe":
        return cls({k: v / 127.0 for k, v in amax.items()}, architecture(cfg))

    def subset(self, names) -> "W8A8Recipe":
        """The recipe restricted to `names` (each must be in this recipe)."""
        names = list(names)
        missing = [n for n in names if n not in self.scales]
        if missing:
            raise ValueError(f"W8A8 recipe has no scale for layer {missing[0]!r}")
        return W8A8Recipe({n: self.scales[n] for n in names}, self.arch)

    def __len__(self):
        return len(self.scales)

    def __contains__(self, name):
        return name in self.scales

    def to_json(self) -> dict:
        return {"format": "b200sd-w8a8", "version": 1, "architecture": self.arch, "activation_scales": self.scales}

    def save(self, path):
        with open(path, "w") as f:
            json.dump(self.to_json(), f, indent=1, sort_keys=True)

    @classmethod
    def load(cls, path) -> "W8A8Recipe":
        with open(path) as f:
            d = json.load(f)
        if d.get("format") != "b200sd-w8a8" or "activation_scales" not in d:
            raise ValueError(f"{path}: not a W8A8 recipe (format b200sd-w8a8)")
        return cls(d["activation_scales"], d.get("architecture"))

    def validate(self, cfg: dict) -> "dict[str, int]":
        """Checks the recipe against the UNet it is applied to; returns the quantized layers -> input channels.
        Raises ValueError naming the layer (or the architecture field) that does not fit."""
        layers = quantizable_layers(cfg)
        if self.arch is not None:
            mine = architecture(cfg)
            for k in _ARCH_KEYS:
                if k in self.arch and self.arch[k] != mine[k]:
                    raise ValueError(f"W8A8 recipe was calibrated for {k}={self.arch[k]}, this UNet has {mine[k]}")
        for name, s in self.scales.items():
            if not _ELIGIBLE.match(name):
                raise ValueError(f"W8A8 recipe layer {name!r} is not a quantizable layer (ResNet conv1 / conv2 or an "
                                 "up-sampler convolution)")
            if name not in layers:
                raise ValueError(f"W8A8 recipe layer {name!r} does not exist in this UNet")
            if not (math.isfinite(s) and s > 0):
                raise ValueError(f"W8A8 recipe layer {name!r} has activation scale {s} (must be finite and > 0)")
            if layers[name] % 16:
                raise ValueError(f"W8A8 recipe layer {name!r} has {layers[name]} input channels (the int8 convolution "
                                 "needs a multiple of 16)")
        return {n: layers[n] for n in self.scales}


def as_recipe(r) -> "W8A8Recipe | None":
    """A recipe, a path to a saved one, or None."""
    if r is None or isinstance(r, W8A8Recipe):
        return r
    return W8A8Recipe.load(r)


def select_from_sensitivity(sensitivity, conv_psnr: float, calibration: W8A8Recipe):
    """Reads the reference's sensitivity JSON ({"conv": {name: psnr}, "einsum": {...}, "model_version": ...}; a path or
    the parsed dict) and keeps the convolutions whose PSNR is >= conv_psnr, as the reference's recipe step does.
    Returns (recipe with those layers' scales from `calibration`, sorted list of every other named layer: kept fp16,
    including the names this engine never quantizes: attention einsums, 1x1 projections, ...)."""
    if not isinstance(sensitivity, dict):
        with open(sensitivity) as f:
            sensitivity = json.load(f)
    if "conv" not in sensitivity:
        raise ValueError("sensitivity JSON has no 'conv' section")
    chosen, kept = [], []
    for name, psnr in sensitivity.get("conv", {}).items():
        (chosen if (_ELIGIBLE.match(name) and float(psnr) >= conv_psnr) else kept).append(name)
    kept += list(sensitivity.get("einsum", {}))
    return calibration.subset(chosen), sorted(kept)


def compute_psnr(a: torch.Tensor, b: torch.Tensor) -> float:
    """PSNR of b against the reference a, with the formula of oracle.restated.compute_psnr."""
    a, b = a.double().flatten(), b.double().flatten()
    mse = ((a - b) ** 2).mean()
    return float(20 * torch.log10((b.abs().max() + 1e-5) / (mse.sqrt() + 1e-10)))
