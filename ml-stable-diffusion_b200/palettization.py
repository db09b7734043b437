"""Weight palettization of the UNet: every large ``nn.Linear`` / ``nn.Conv2d`` weight stored as n-bit indices into one
per-tensor palette (lookup table, LUT) of 2^n fp16 values, decoded in the GEMM / convolution kernel's producer
(``lib.linear`` / ``lib.conv3x3`` with a :class:`PalettizedWeight`, ``b200sd_gemm_lut``).

Semantics (restated from the reference's ``mixed_bit_compression_pre_analysis.py`` / ``mixed_bit_compression_apply.py``
and ``torch2coreml.py --quantize-nbits``; not bit-parity with coremltools' k-means):
  * eligible layers: every Linear / Conv2d of the diffusers UNet whose weight has more than 1e5 elements
    (``get_palettizable_modules``);
  * a recipe maps eligible layers to 1, 2, 4, 6, 8 or 16 bits (16: keep fp16); unnamed layers stay fp16;
  * palette: deterministic 1-D k-means over the histogram of the tensor's distinct fp16 values -- weighted Lloyd
    iterations from a quantile (and a uniform-grid) initialisation, no RNG.  When 2^n >= the number of distinct values the palette is those
    values (exact).  Entries are rounded to fp16 and every weight takes its nearest rounded entry, ties to the lower
    index;
  * ``decoded_state_dict`` is the reference's ``fake_palette_from_recipe``: each palettized weight replaced by
    ``LUT[idx]``.
"""
from __future__ import annotations

import json
import math

import torch

from . import config as _config

NBITS = (1, 2, 4, 6, 8)
ALLOWED_NBITS = NBITS + (16,)
MIN_SIZE = 100_000  # the reference's PALETTIZE_MIN_SIZE
_LLOYD_ITERS = 100


def palettizable_layers(cfg: dict) -> "dict[str, int]":
    """Every eligible layer of a UNet config -> its weight's element count, in state-dict (module) order."""
    out = {}
    for key, shape in _config.unet_param_shapes(cfg).items():
        if key.endswith(".weight") and len(shape) in (2, 4) and math.prod(shape) > MIN_SIZE:
            out[key[: -len(".weight")]] = math.prod(shape)
    return out


def _linear_and_conv_layers(cfg):
    return {k[: -len(".weight")] for k, s in _config.unet_param_shapes(cfg).items() if k.endswith(".weight") and len(s) in (2, 4)}


def as_recipe(palettization, cfg: dict):
    """A palettization argument -> {layer: nbits} of the layers that are palettized (16-bit entries dropped), or None.

    Accepts an int (every eligible layer at that width, like ``--quantize-nbits``), a {layer: nbits} dict, or
    (path, recipe_key) into a pre-analysis JSON (read from ``["recipes"][recipe_key]``).  Raises ValueError naming the
    layer for an unknown or ineligible layer or an illegal width, and naming the available keys for an unknown key."""
    if palettization is None:
        return None
    layers = palettizable_layers(cfg)
    if isinstance(palettization, bool):
        raise ValueError(f"palettization: expected nbits, a {{layer: nbits}} dict or (json path, recipe key), got {palettization!r}")
    if isinstance(palettization, int):
        if palettization not in ALLOWED_NBITS:
            raise ValueError(f"palettization: nbits={palettization} is not one of {ALLOWED_NBITS}")
        recipe = {name: palettization for name in layers}
    elif isinstance(palettization, (tuple, list)) and len(palettization) == 2:
        path, key = palettization
        with open(path) as f:
            data = json.load(f)
        recipes = data.get("recipes") if isinstance(data, dict) else None
        if not isinstance(recipes, dict):
            raise ValueError(f"palettization: {path} has no 'recipes' table")
        if key not in recipes:
            raise ValueError(f"palettization: recipe key {key!r} is not in {path}; available recipes: {sorted(recipes)}")
        recipe = dict(recipes[key])
    elif isinstance(palettization, dict):
        recipe = dict(palettization)
    else:
        raise ValueError(f"palettization: expected nbits, a {{layer: nbits}} dict or (json path, recipe key), got {palettization!r}")
    known = None
    for name, nbits in recipe.items():
        if name not in layers:
            known = known if known is not None else _linear_and_conv_layers(cfg)
            if name in known:
                raise ValueError(f"palettization: layer {name} is not eligible (weight of at most {MIN_SIZE} elements)")
            raise ValueError(f"palettization: unknown layer {name}")
        if isinstance(nbits, bool) or nbits not in ALLOWED_NBITS:
            raise ValueError(f"palettization: layer {name}: nbits={nbits!r} is not one of {ALLOWED_NBITS}")
    return {name: int(n) for name, n in recipe.items() if n != 16}


def nominal_bits(recipe: dict, cfg: dict) -> float:
    """Average bits per eligible weight a recipe asks for (16 for layers it leaves fp16)."""
    layers = palettizable_layers(cfg)
    return sum(recipe.get(k, 16) * n for k, n in layers.items()) / sum(layers.values())


# ------------------------------------------------------------------------------------------------ palette fitting
def _nearest(values, lut):
    """Index of the nearest entry of the ascending fp16-valued `lut` (float64) for each value; ties to the lower index."""
    i = torch.searchsorted(lut, values).clamp(1, lut.numel() - 1)
    lo, hi = lut[i - 1], lut[i]
    return torch.where((values - lo).abs() <= (hi - values).abs(), i - 1, i)


def _lloyd(v, c, centres):
    """Weighted Lloyd iterations over the ascending distinct values v with counts c.  Each cluster is the run of values
    between the midpoints of its neighbours (a value on a midpoint goes to the lower centre, as in _nearest), so one
    iteration is a binary search of the k - 1 midpoints and two prefix-sum differences."""
    s1 = torch.cat([torch.zeros(1, dtype=torch.float64), torch.cumsum(v * c, 0)])
    s0 = torch.cat([torch.zeros(1, dtype=torch.float64), torch.cumsum(c, 0)])
    for _ in range(_LLOYD_ITERS):
        centres, _ = torch.sort(centres)
        mid = (centres[:-1] + centres[1:]) * 0.5
        ends = torch.cat([torch.zeros(1, dtype=torch.long), torch.searchsorted(v, mid, right=True),
                          torch.full((1,), v.numel(), dtype=torch.long)])
        n = s0[ends[1:]] - s0[ends[:-1]]
        new = torch.where(n > 0, (s1[ends[1:]] - s1[ends[:-1]]) / n.clamp(min=1e-300), centres)
        if torch.equal(new, centres):
            break
        centres = new
    return torch.sort(centres)[0]


def fit_palette(w: torch.Tensor, nbits: int):
    """(lut fp16 [2^nbits] ascending, idx uint8 with w's shape): the palette of `w` (rounded to fp16 first).

    Lloyd's algorithm on the histogram of the distinct values, started from the weighted quantiles (i + 0.5) / 2^n
    and from the uniform grid over [min, max]; the run with the lower weighted squared error wins, an empty cluster
    keeps its centre.  Runs on w's device for the histogram and the assignment, on the CPU in float64
    for the iterations (a few thousand distinct values at most 65536), so the result does not depend on the device."""
    if nbits not in NBITS:
        raise ValueError(f"fit_palette: nbits={nbits} is not one of {NBITS}")
    k = 1 << nbits
    vals, inv, counts = torch.unique(w.detach().half().reshape(-1), return_inverse=True, return_counts=True)
    v = vals.double().cpu()
    c = counts.double().cpu()
    if v.numel() <= k:
        centres = torch.cat([v, v[-1:].expand(k - v.numel())])
    else:
        cdf = torch.cumsum(c, 0) / c.sum()
        q = (torch.arange(k, dtype=torch.float64) + 0.5) / k
        best = None
        # Lloyd from the quantiles, and from the uniform grid over [min, max] (so the result is never worse than it)
        for init in (v[torch.searchsorted(cdf, q).clamp(max=v.numel() - 1)], torch.linspace(float(v[0]), float(v[-1]), k,
                                                                                          dtype=torch.float64)):
            cen = _lloyd(v, c, init)
            sse = float((c * (v - cen[_nearest(v, cen)]) ** 2).sum())
            if best is None or sse < best[0]:
                best = (sse, cen)
        centres = best[1]
    lut = torch.sort(centres.half())[0]
    vidx = _nearest(v, lut.double()).to(torch.uint8)
    idx = vidx.to(w.device)[inv].reshape(w.shape)
    return lut, idx


def decode(lut: torch.Tensor, idx: torch.Tensor) -> torch.Tensor:
    return lut.to(idx.device)[idx.long()]


# ------------------------------------------------------------------------------------------------ packing
def row_bytes(k: int, nbits: int) -> int:
    """Bytes per packed row of k indices (a multiple of 16, the TMA row-stride granularity)."""
    return (k * nbits + 127) // 128 * 16


def pack_indices(idx: torch.Tensor, nbits: int) -> torch.Tensor:
    """[N, K] indices (K a multiple of 64) -> uint8 [N, row_bytes]: each row a little-endian bit stream, index k at bits
    [k * nbits, (k + 1) * nbits).  The layout does not depend on the kernel's tile width."""
    n, k = idx.shape
    bits = (idx.to(torch.uint8).unsqueeze(-1) >> torch.arange(nbits, dtype=torch.uint8, device=idx.device)) & 1
    bits = bits.reshape(n, k * nbits // 8, 8)
    by = torch.zeros(n, k * nbits // 8, dtype=torch.uint8, device=idx.device)
    for b in range(8):
        by |= bits[:, :, b] << b
    out = torch.zeros(n, row_bytes(k, nbits), dtype=torch.uint8, device=idx.device)
    out[:, : by.shape[1]] = by
    return out


def unpack_indices(packed: torch.Tensor, nbits: int, k: int) -> torch.Tensor:
    """Inverse of pack_indices: uint8 [N, K] indices."""
    n = packed.shape[0]
    by = packed[:, : k * nbits // 8]
    bits = (by.unsqueeze(-1) >> torch.arange(8, dtype=torch.uint8, device=packed.device)) & 1
    bits = bits.reshape(n, k, nbits)
    idx = torch.zeros(n, k, dtype=torch.uint8, device=packed.device)
    for b in range(nbits):
        idx |= bits[:, :, b] << b
    return idx


class PalettizedWeight:
    """A GEMM / convolution weight held as packed n-bit indices and up to three row-segment palettes.

    packed uint8 [N, row_bytes] (the 2-D weight's columns in the kernel's k order), lut fp16 [3, 256], nbits the
    container width, seg_ends the first rows of segments 1 and 2, kscale an optional fp32 per-k scale (a folded
    LayerNorm's gamma), stored_bits / nominal the container and recipe widths per segment."""

    def __init__(self, packed, lut, nbits, k, seg_ends=None, kscale=None, nominal=None):
        self.packed, self.lut, self.nbits, self.k = packed, lut, nbits, k
        n = packed.shape[0]
        self.seg_ends = tuple(seg_ends) if seg_ends is not None else (n, n)
        self.kscale = kscale
        self.nominal = nominal if nominal is not None else (nbits,)
        self.layers = []  # the recipe layers whose rows this weight holds (UNetEngine sets them)
        self.shape = (n, k)
        self.dtype = torch.float16

    @property
    def device(self):
        return self.packed.device

    def tensors(self):
        """The device tensors this weight owns (kscale is the caller's: the engine's LayerNorm gamma)."""
        yield self.packed
        yield self.lut

    def decoded(self) -> torch.Tensor:
        """The fp16 [N, K] weight the kernel computes with (for tests and the oracle)."""
        idx = unpack_indices(self.packed, self.nbits, self.k).long()
        seg = torch.zeros(self.shape[0], dtype=torch.long, device=idx.device)
        seg[self.seg_ends[0]:] += 1
        seg[self.seg_ends[1]:] += 1
        w = self.lut.to(idx.device)[seg[:, None], idx]
        if self.kscale is not None:
            w = (w.float() * self.kscale.to(idx.device)[None, :]).half()
        return w


def palettized(segments, kscale=None) -> PalettizedWeight:
    """[(lut fp16 [2^n], idx [n_s, K] in the kernel's k order, nbits)] of one launch's row segments (one to three, same
    K) -> its PalettizedWeight.  The segments share the largest width as container."""
    if not 1 <= len(segments) <= 3:
        raise ValueError("palettized: one to three row segments")
    nb = max(n for _, _, n in segments)
    dev = segments[0][1].device
    lut = torch.zeros(3, 256, dtype=torch.float16, device=dev)
    ends, off = [], 0
    for s, (l, i, _) in enumerate(segments):
        lut[s, : l.numel()] = l.to(dev)
        off += i.shape[0]
        ends.append(off)
    ends = (ends[:2] + [off, off])[:2] if len(ends) > 1 else [off, off]
    idx = torch.cat([i for _, i, _ in segments], 0)
    return PalettizedWeight(pack_indices(idx, nb), lut, nb, idx.shape[1], seg_ends=ends,
                            kscale=None if kscale is None else kscale.to(device=dev, dtype=torch.float32).contiguous(),
                            nominal=tuple(n for _, _, n in segments))


def decoded_state_dict(sd: dict, recipe, cfg: dict = None) -> dict:
    """The state dict with every palettized weight replaced by LUT[idx] in fp16 (the reference's
    ``fake_palette_from_recipe``).  recipe: {layer: nbits} (or anything as_recipe accepts, with cfg)."""
    if not isinstance(recipe, dict) or cfg is not None:
        recipe = as_recipe(recipe, cfg)
    out = dict(sd)
    for name, nbits in (recipe or {}).items():
        if nbits == 16:
            continue
        w = sd[name + ".weight"]
        lut, idx = fit_palette(w, nbits)
        out[name + ".weight"] = decode(lut, idx).to(dtype=torch.float16).reshape(w.shape)
    return out
