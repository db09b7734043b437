"""W8A8 quantization of the UNet's ResNet and up-sampler 3x3 convolutions (int8 weights and activations on the int8
wgmma kernel, ``lib.conv3x3_s8``) and, opted in through a separate section of the recipe, of its transformers' linear
projections (``lib.linear_s8``).

Semantics (restated from the reference's ``activation_quantization.py``; not bit-parity with coremltools):
  * weights: symmetric int8 per output channel, s_w[n] = max_k |W[n, k]| / 127 (an all-zero row gets scale 1),
    q = clamp(rne(W / s_w), -127, 127);
  * activations: symmetric int8 per tensor, s_a = amax / 127, where amax is max |x| at the layer's input over every UNet
    call of a calibration run with the fp16 engine (``B200StableDiffusionPipeline.calibrate_unet``).  For a ResNet
    convolution x is the GroupNorm + SiLU output, for an up-sampler convolution the tensor before the upsample.  For
    the linear layers (``quantizable_linear_layers``) x is what the reference's layer sees: the GroupNorm output for
    proj_in, the norm1 / norm2 / norm3 LayerNorm output for attn1.to_q|k|v / attn2.to_q / ff.net.0.proj, the GEGLU
    output for ff.net.2 and the last transformer block's output for proj_out;
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
# transformer linears the engine can run in W8A8.  attn1's to_q / to_k / to_v share one input and one launch, so a recipe
# names all three with one scale or none of them (the reference may quantize them one at a time)
_ATTN = r"(down_blocks\.\d+\.attentions\.\d+|mid_block\.attentions\.0|up_blocks\.\d+\.attentions\.\d+)"
_ELIGIBLE_LINEAR = re.compile(rf"^{_ATTN}\.(proj_in|proj_out|transformer_blocks\.\d+\."
                              r"(attn1\.to_[qkv]|attn2\.to_q|ff\.net\.0\.proj|ff\.net\.2))$")
# linears the engine never quantizes, with the reason the validator gives
_NOT_LINEAR = (
    (re.compile(r"\.to_out\.0$"), "attention output projections (to_out.0) stay fp16, as the reference's recipe keeps them"),
    (re.compile(r"\.attn2\.to_[kv]$"), "cross-attention to_k / to_v run once per prompt, not per step"),
    (re.compile(r"(\.conv_shortcut|\.downsamplers\.0\.conv|^conv_in|^conv_out|time_emb_proj|^time_embedding\.|"
                r"^add_embedding\.)"), "shortcuts, down-samplers, conv_in / conv_out and time-embedding projections stay fp16"),
)


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


def _transformers(cfg: dict):
    """(transformer prefix, channels, depth) of every transformer of a UNet config, in launch order."""
    boc = list(cfg["block_out_channels"])
    nb, lpb = len(boc), cfg.get("layers_per_block", 2)
    tl = cfg.get("transformer_layers_per_block", 1)
    depth = list(tl) if isinstance(tl, (list, tuple)) else [tl] * nb
    out = []
    for i, typ in enumerate(cfg["down_block_types"]):
        if typ == "CrossAttnDownBlock2D":
            out += [(f"down_blocks.{i}.attentions.{j}", boc[i], depth[i]) for j in range(lpb)]
    out.append(("mid_block.attentions.0", boc[-1], cfg.get("mid_block_transformer_layers", depth[-1])))
    for i, typ in enumerate(cfg["up_block_types"]):
        if typ == "CrossAttnUpBlock2D":
            out += [(f"up_blocks.{i}.attentions.{j}", boc[::-1][i], depth[::-1][i]) for j in range(lpb + 1)]
    return out


def quantizable_linear_layers(cfg: dict) -> "dict[str, int]":
    """Every transformer linear this engine can run in W8A8 for a UNet config -> its input channel count, in launch
    order: proj_in, per block attn1.to_q / to_k / to_v, attn2.to_q, ff.net.0.proj, ff.net.2, then proj_out.  (SD 1.x's
    1x1-convolution proj_in / proj_out are the same matrices.)"""
    out = {}
    for p, c, depth in _transformers(cfg):
        out[p + ".proj_in"] = c
        for d in range(depth):
            b = f"{p}.transformer_blocks.{d}"
            for n in ("attn1.to_q", "attn1.to_k", "attn1.to_v", "attn2.to_q", "ff.net.0.proj"):
                out[f"{b}.{n}"] = c
            out[f"{b}.ff.net.2"] = 4 * c
        out[p + ".proj_out"] = c
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
    were calibrated on.  `scales` holds the convolutions (quantizable_layers), `linear_scales` the transformer linears
    (quantizable_linear_layers), a separate section that only recipes calibrated or selected with linear=True fill."""

    def __init__(self, scales: "dict[str, float]", arch: "dict | None" = None,
                 linear_scales: "dict[str, float] | None" = None):
        self.scales = {str(k): float(v) for k, v in scales.items()}
        self.arch = arch
        self.linear_scales = {str(k): float(v) for k, v in (linear_scales or {}).items()}

    @classmethod
    def from_amax(cls, amax: "dict[str, float]", cfg: dict, linear_amax: "dict[str, float] | None" = None) -> "W8A8Recipe":
        return cls({k: v / 127.0 for k, v in amax.items()}, architecture(cfg),
                   {k: v / 127.0 for k, v in (linear_amax or {}).items()})

    def subset(self, names, linear_names=()) -> "W8A8Recipe":
        """The recipe restricted to the convolutions `names` and the linears `linear_names` (each must be in it)."""
        names, linear_names = list(names), list(linear_names)
        missing = [n for n in names if n not in self.scales] + [n for n in linear_names if n not in self.linear_scales]
        if missing:
            raise ValueError(f"W8A8 recipe has no scale for layer {missing[0]!r}")
        return W8A8Recipe({n: self.scales[n] for n in names}, self.arch, {n: self.linear_scales[n] for n in linear_names})

    def __len__(self):
        return len(self.scales)

    def __contains__(self, name):
        return name in self.scales

    def to_json(self) -> dict:
        d = {"format": "b200sd-w8a8", "version": 1, "architecture": self.arch, "activation_scales": self.scales}
        if self.linear_scales:
            d["version"] = 2
            d["linear_activation_scales"] = self.linear_scales
        return d

    def save(self, path):
        with open(path, "w") as f:
            json.dump(self.to_json(), f, indent=1, sort_keys=True)

    @classmethod
    def load(cls, path) -> "W8A8Recipe":
        with open(path) as f:
            d = json.load(f)
        if d.get("format") != "b200sd-w8a8" or "activation_scales" not in d:
            raise ValueError(f"{path}: not a W8A8 recipe (format b200sd-w8a8)")
        return cls(d["activation_scales"], d.get("architecture"), d.get("linear_activation_scales"))

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
        self.validate_linear(cfg)
        return {n: layers[n] for n in self.scales}

    def validate_linear(self, cfg: dict) -> "dict[str, int]":
        """Checks the linear section against the UNet; returns the quantized linears -> input channels.  Raises
        ValueError naming the layer that does not fit."""
        layers = quantizable_linear_layers(cfg)
        for name, s in self.linear_scales.items():
            for pat, why in _NOT_LINEAR:
                if pat.search(name):
                    raise ValueError(f"W8A8 recipe linear layer {name!r} is not quantizable: {why}")
            if not _ELIGIBLE_LINEAR.match(name):
                raise ValueError(f"W8A8 recipe linear layer {name!r} is not a quantizable linear (proj_in / proj_out, "
                                 "attn1.to_q|k|v, attn2.to_q, ff.net.0.proj, ff.net.2)")
            if name not in layers:
                raise ValueError(f"W8A8 recipe linear layer {name!r} does not exist in this UNet")
            if not (math.isfinite(s) and s > 0):
                raise ValueError(f"W8A8 recipe linear layer {name!r} has activation scale {s} (must be finite and > 0)")
            if layers[name] % 16:
                raise ValueError(f"W8A8 recipe linear layer {name!r} has {layers[name]} input channels (the int8 GEMM "
                                 "needs a multiple of 16)")
            if ".attn1.to_" in name:
                block = name.rsplit(".", 1)[0]
                triple = [f"{block}.to_{n}" for n in "qkv"]
                absent = [n for n in triple if n not in self.linear_scales]
                if absent:
                    raise ValueError(f"W8A8 recipe linear layer {absent[0]!r} is missing: attn1.to_q / to_k / to_v run "
                                     f"as one launch on one input, so they are quantized together (got {name!r})")
                if len({self.linear_scales[n] for n in triple}) != 1:
                    raise ValueError(f"W8A8 recipe linear layer {name!r}: attn1.to_q / to_k / to_v share one input and "
                                     "need one activation scale")
        return {n: layers[n] for n in self.linear_scales}


def as_recipe(r) -> "W8A8Recipe | None":
    """A recipe, a path to a saved one, or None."""
    if r is None or isinstance(r, W8A8Recipe):
        return r
    return W8A8Recipe.load(r)


def select_from_sensitivity(sensitivity, conv_psnr: float, calibration: W8A8Recipe, linear: bool = False):
    """Reads the reference's sensitivity JSON ({"conv": {name: psnr}, "einsum": {...}, "model_version": ...}; a path or
    the parsed dict) and keeps the convolutions whose PSNR is >= conv_psnr, as the reference's recipe step does.
    linear: the same threshold also selects the eligible transformer linears (the reference's UNet runs them as 1x1
    convolutions, so they are in its "conv" section); an attn1 to_q / to_k / to_v triple is kept only when all three
    pass, and to_out.0 never is.
    Returns (recipe with those layers' scales from `calibration`, sorted list of every other named layer: kept fp16,
    including the names this engine never quantizes: attention einsums, 1x1 projections, ...)."""
    if not isinstance(sensitivity, dict):
        with open(sensitivity) as f:
            sensitivity = json.load(f)
    if "conv" not in sensitivity:
        raise ValueError("sensitivity JSON has no 'conv' section")
    conv = {name: float(psnr) for name, psnr in sensitivity.get("conv", {}).items()}
    chosen, chosen_lin, kept = [], [], []
    for name, psnr in conv.items():
        if _ELIGIBLE.match(name) and psnr >= conv_psnr:
            chosen.append(name)
        elif linear and _ELIGIBLE_LINEAR.match(name) and psnr >= conv_psnr:
            if ".attn1.to_" in name:
                block = name.rsplit(".", 1)[0]
                if not all(conv.get(f"{block}.to_{n}", -math.inf) >= conv_psnr for n in "qkv"):
                    kept.append(name)
                    continue
            chosen_lin.append(name)
        else:
            kept.append(name)
    kept += list(sensitivity.get("einsum", {}))
    return calibration.subset(chosen, chosen_lin), sorted(kept)


def compute_psnr(a: torch.Tensor, b: torch.Tensor) -> float:
    """PSNR of b against the reference a, with the formula of oracle.restated.compute_psnr."""
    a, b = a.double().flatten(), b.double().flatten()
    mse = ((a - b) ** 2).mean()
    return float(20 * torch.log10((b.abs().max() + 1e-5) / (mse.sqrt() + 1e-10)))
