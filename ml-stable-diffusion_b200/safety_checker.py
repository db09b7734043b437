"""Stable Diffusion safety checker on the sm_90a kernels.

Replaces the ``safety_checker`` Core ML model of the reference and the host preprocessing in front of it
(``pipeline.py:286-311``: ``feature_extractor(numpy_to_pil(image))``, then ``safety_checker(clip_input, images,
adjustment)``).  The network is diffusers' ``StableDiffusionSafetyChecker`` as the reference converts it
(``forward_coreml``, ``torch2coreml.py:1177-1209``):

* CLIP preprocessing (``csrc/vision.cu``): Pillow's BICUBIC shortest-edge resize in its 8-bit fixed-point form, centre
  crop, rescale and normalise -- bit-identical to transformers 4.44.2's ``CLIPImageProcessor`` on ``numpy_to_pil``'s
  images, which ``image_postprocess(want_u8=True)`` already produces on the device;
* the ``CLIPVisionModel`` tower: patch extraction + one patch-embedding GEMM that also adds the position embeddings
  (the class token's row of the GEMM operand is zero, its residual row is ``class_embedding + position_embedding[0]``),
  ``pre_layrnorm``, the shared pre-LN encoder (``clip_encoder``, non-causal, 257 tokens), ``post_layernorm`` of the
  class token, the visual projection;
* concept scoring against the L2-normalised concept tables and the blacking out of flagged images.
"""
from __future__ import annotations

import math

import numpy as np
import torch
import torch.nn.functional as F

from . import clip_encoder as E
from . import config as C
from . import lib as L
from .model import B200Model


def _bicubic(x):
    """Pillow's bicubic filter (Resample.c, a = -0.5), with its exact operation order."""
    a = -0.5
    x = abs(x)
    if x < 1.0:
        return ((a + 2.0) * x - (a + 3.0)) * x * x + 1
    if x < 2.0:
        return (((x - 5) * x + 8) * x - 4) * a
    return 0.0


def resample_table(in_size: int, out_size: int):
    """Pillow's BICUBIC coefficients for resizing ``in_size`` samples to ``out_size`` (``precompute_coeffs`` +
    ``normalize_coeffs_8bpc``, float64): -> (bounds int32 [out_size, 2] = (first input index, taps), coeffs int32
    [out_size, ksize], the weights with 22 fractional bits, rounded half away from zero)."""
    scale = in_size / out_size
    fs = max(scale, 1.0)
    support = 2.0 * fs
    ss = 1.0 / fs
    ksize = int(math.ceil(support)) * 2 + 1
    bounds = np.zeros((out_size, 2), np.int32)
    coeffs = np.zeros((out_size, ksize), np.int32)
    for i in range(out_size):
        center = (i + 0.5) * scale
        xmin = max(int(center - support + 0.5), 0)
        n = min(int(center + support + 0.5), in_size) - xmin
        w = [_bicubic((j + xmin - center + 0.5) * ss) for j in range(n)]
        total = 0.0
        for v in w:  # sequential, as Pillow sums (Python's sum() is compensated)
            total += v
        for j, v in enumerate(w):
            v = v / total if total != 0.0 else v
            coeffs[i, j] = int(v * (1 << 22) + 0.5) if v >= 0 else int(-0.5 + v * (1 << 22))
        bounds[i] = (xmin, n)
    return bounds, coeffs


def resize_shape(h: int, w: int, size: int):
    """transformers' ``get_resize_output_image_size(default_to_square=False)``: the shortest edge becomes ``size``, the
    long edge ``int(size * long / short)``.  -> (new_h, new_w)."""
    short, long = (w, h) if w <= h else (h, w)
    new_long = int(size * long / short)
    return (new_long, size) if w <= h else (size, new_long)


class SafetyCheckerEngine:
    """``cfg``: ``config.SD_SAFETY_CHECKER`` or ``config.safety_checker_config(config.json)``; ``state_dict``: the
    ``safety_checker`` schema of ``checkpoint``; ``preprocessor_cfg``: ``checkpoint.preprocessor_config(...)`` (None:
    CLIPImageProcessor's defaults)."""

    def __init__(self, cfg: dict, state_dict: dict, preprocessor_cfg=None, device="cuda"):
        from .checkpoint import PREPROCESS_DEFAULTS
        L.load()
        self.cfg = dict(C.CLIP_VISION_DEFAULTS, **cfg)
        cfg = self.cfg
        self.dev = torch.device(device)
        self.d, self.heads = cfg["hidden_size"], cfg["num_attention_heads"]
        if self.d // self.heads != 64 or self.d % self.heads:
            raise L.B200SDError(f"safety checker head dim {self.d / self.heads:g} not supported by the attention kernel (64)")
        if cfg["hidden_act"] not in E.ACT:
            raise L.B200SDError(f"unsupported hidden_act {cfg['hidden_act']!r}")
        self.act = E.ACT[cfg["hidden_act"]]
        self.eps = cfg["layer_norm_eps"]
        self.image_size, self.patch, self.channels = cfg["image_size"], cfg["patch_size"], cfg["num_channels"]
        if self.image_size % self.patch or self.channels != 3:
            raise L.B200SDError(f"image_size {self.image_size} / patch_size {self.patch} / {self.channels} channels: the "
                                "vision tower needs whole patches of RGB images")
        self.tokens = (self.image_size // self.patch) ** 2 + 1
        self.k = self.channels * self.patch * self.patch
        self.k_pad = (self.k + 7) // 8 * 8  # the GEMM reads rows of whole 16-byte vectors
        self.pre = dict(preprocessor_cfg or PREPROCESS_DEFAULTS)
        if (self.pre["crop_h"], self.pre["crop_w"]) != (self.image_size, self.image_size):
            raise ValueError(f"the feature extractor crops {self.pre['crop_h']}x{self.pre['crop_w']}, the vision tower "
                             f"reads {self.image_size}x{self.image_size}")
        self._pack(state_dict)
        self._tables = {}
        self._pos_rows = {}

    def _pack(self, sd):
        dev, d = self.dev, self.d
        v = "vision_model.vision_model."

        def f16(t):
            return t.detach().to(device=dev, dtype=torch.float16).contiguous()

        def f32(t):
            return t.detach().to(device=dev, dtype=torch.float32).contiguous()

        w = torch.zeros(d, self.k_pad, dtype=torch.float32)
        w[:, :self.k] = sd[v + "embeddings.patch_embedding.weight"].detach().float().reshape(d, self.k)
        pos = sd[v + "embeddings.position_embedding.weight"].detach().float().clone()
        pos[0] += sd[v + "embeddings.class_embedding"].detach().float()  # the class token's embedding row
        self.w = {
            "patch": f16(w), "pos": f16(pos),
            "pre_g": f32(sd[v + "pre_layrnorm.weight"]), "pre_b": f32(sd[v + "pre_layrnorm.bias"]),
            "layers": E.pack_layers(sd, v + "encoder.layers.", self.cfg["num_hidden_layers"], dev),
            "post_g": f32(sd[v + "post_layernorm.weight"]), "post_b": f32(sd[v + "post_layernorm.bias"]),
            "proj": f16(sd["visual_projection.weight"]),
        }
        self.set_concepts(sd)

    def set_concepts(self, sd):
        """(Re)load the concept tables from ``sd``'s concept_embeds, special_care_embeds and their _weights (fp32).
        The rows are L2-normalised here once: F.normalize(text_embeds) of cosine_distance is constant."""
        def f32(t):
            return t.detach().to(device=self.dev, dtype=torch.float32).contiguous()

        self.w.update(concepts=f32(F.normalize(sd["concept_embeds"].detach().float(), dim=1)),
                      concept_w=f32(sd["concept_embeds_weights"]),
                      special=f32(F.normalize(sd["special_care_embeds"].detach().float(), dim=1)),
                      special_w=f32(sd["special_care_embeds_weights"]))

    # -- stages ------------------------------------------------------------------------------------------------------
    def tables(self, h, w):
        """Device resampling tables of an h x w image, restricted to the rows / columns the centre crop keeps."""
        key = (h, w)
        t = self._tables.get(key)
        if t is None:
            size, ch, cw = self.pre["size"], self.pre["crop_h"], self.pre["crop_w"]
            nh, nw = resize_shape(h, w, size)
            top, left = (nh - ch) // 2, (nw - cw) // 2
            hb, hc = resample_table(w, nw)
            vb, vc = resample_table(h, nh)
            as_dev = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(self.dev)  # noqa: E731
            t = ((as_dev(hb[left:left + cw]), as_dev(hc[left:left + cw])),
                 (as_dev(vb[top:top + ch]), as_dev(vc[top:top + ch])))
            self._tables[key] = t
        return t

    def preprocess(self, images_u8):
        """u8 NHWC [n, h, w, 3] (``numpy_to_pil``'s pixels) -> fp32 pixel_values [n, 3, S, S]."""
        _, h, w, _ = images_u8.shape
        ht, vt = self.tables(h, w)
        return L.clip_preprocess(images_u8, ht, vt, self.pre["mean"], self.pre["std"])

    def _positions(self, n):
        """[n * tokens, d] fp16 residual of the patch GEMM: per image the class token's embedding, then the position
        embeddings of the patches."""
        t = self._pos_rows.get(n)
        if t is None:
            t = self.w["pos"].repeat(n, 1).contiguous()
            self._pos_rows[n] = t
        return t

    def tower(self, pixel_values):
        """fp32 pixel_values [n, 3, S, S] -> (image_embeds fp32 [n, projection_dim], the encoder's last hidden state
        fp16 [n * tokens, d] before post_layernorm)."""
        w, n, d = self.w, pixel_values.shape[0], self.d
        a = L.patchify(pixel_values, self.patch, self.k_pad)
        x = L.linear(a, w["patch"], None, self._positions(n), static_w=True)
        x = L.layer_norm(x, w["pre_g"], w["pre_b"], eps=self.eps)
        x = E.run_layers(x, w["layers"], n, self.tokens, d, self.heads, self.act, self.eps, causal=False)
        cls = x.view(n, self.tokens, d)[:, 0].contiguous()
        pooled = L.layer_norm(cls, w["post_g"], w["post_b"], eps=self.eps)
        return L.linear_small(pooled.float(), w["proj"]), x

    def concepts(self, image_embeds, adjustment=None):
        """-> (concept_scores fp32 [n, 17], has_nsfw fp32 [n])."""
        w = self.w
        return L.safety_concepts(image_embeds, w["concepts"], w["concept_w"], w["special"], w["special_w"], adjustment)

    def check(self, images=None, images_u8=None, pixel_values=None, adjustment=None):
        """The whole stage on the device, no host synchronisation: preprocess ``images_u8`` (unless ``pixel_values``
        is given), run the tower and the head, zero the flagged images in place (fp32 ``images`` and / or
        ``images_u8``).  -> (has_nsfw fp32 [n], concept_scores fp32 [n, 17])."""
        if pixel_values is None:
            if images_u8 is None:
                raise ValueError("the safety checker needs images_u8 or pixel_values")
            pixel_values = self.preprocess(images_u8)
        emb, _ = self.tower(pixel_values)
        scores, flags = self.concepts(emb, adjustment)
        if images is not None or images_u8 is not None:
            L.filter_images(flags, images, images_u8)
        return flags, scores


class SafetyCheckerModel(B200Model):
    """``safety_checker(clip_input, images, adjustment)`` with the Core ML model's names (torch2coreml.py:1161-1165,
    :1270): inputs ``clip_input`` fp16 (B, 3, 224, 224), ``images`` fp16 (B, H, W, 3), ``adjustment`` fp16 (1,);
    outputs ``filtered_images`` (B, H, W, 3), ``has_nsfw_concepts`` (B, 1, 1, 1) and ``concept_scores`` (B, 17), fp32."""

    def __init__(self, cfg, state_dict, preprocessor_cfg=None, batch=1, height=512, width=512, device="cuda"):
        self.engine = SafetyCheckerEngine(cfg, state_dict, preprocessor_cfg, device)
        s = self.engine.image_size
        f16 = np.dtype(np.float16)
        spec = {"clip_input": {"shape": (batch, 3, s, s), "dtype": f16},
                "images": {"shape": (batch, height, width, 3), "dtype": f16},
                "adjustment": {"shape": (1,), "dtype": f16}}
        super().__init__(spec, device)
        self.batch = batch
        self._clip = torch.zeros(batch, 3, s, s, dtype=torch.float32, device=self.device)
        self._images = torch.zeros(batch, height, width, 3, dtype=torch.float32, device=self.device)
        self._adj = torch.zeros(1, dtype=torch.float32, device=self.device)

    def __call__(self, **kwargs):
        self._verify_inputs(**kwargs)
        missing = [k for k in self.expected_inputs if k not in kwargs]
        if missing:
            raise ValueError(f"Missing inputs: {missing}")
        as_numpy = isinstance(kwargs["clip_input"], np.ndarray)
        self._to_device(kwargs["clip_input"], self._clip)
        self._to_device(kwargs["images"], self._images)
        self._to_device(kwargs["adjustment"], self._adj)
        flags, scores = self.engine.check(images=self._images, pixel_values=self._clip, adjustment=self._adj)
        out = {"filtered_images": self._images.clone(), "has_nsfw_concepts": flags.reshape(self.batch, 1, 1, 1),
               "concept_scores": scores}
        return {k: v.cpu().numpy() for k, v in out.items()} if as_numpy else out
