"""VAE decoder on the sm_90a kernels (same conv / GroupNorm / GEMM kernels as the UNet).

Replaces the ``vae_decoder`` Core ML model the reference calls once per image
(``pipeline.py:313-320``), whose graph is ``decoder(post_quant_conv(z))`` of diffusers'
``AutoencoderKL`` (``torch2coreml.py:584-594``; architecture restated in SURVEY.md Appendix B1).
NHWC 16-bit activations; the single-head d=512 mid-block attention runs as two tensor-core GEMMs
around a row-softmax kernel (scores fp32), since the flash kernel is specialised for d=64.

The activations are fp16 unless the engine is built with ``dtype=torch.bfloat16``.  bf16 has fp32's exponent
range: it is for the VAEs whose checkpoint sets ``force_upcast`` (the stock SDXL VAE, whose decoder activations
exceed fp16's 65504; diffusers upcasts that VAE to fp32, the reference converts it in FLOAT32).  Then the GEMM /
convolution weights are bf16 and every kernel of the forward runs its bf16 instantiation: each op follows its
input's dtype, and the three ops that read fp32 (latent_prep, nchw_to_nhwc, softmax_rows) write the engine's dtype.
Biases, norm parameters, statistics and accumulators stay fp32 either way.
"""
from __future__ import annotations

import numpy as np
import torch

from . import lib as L
from .model import B200Model
from .unet import _Packer, _w2d


class VAEDecoderEngine:
    def __init__(self, cfg: dict, state_dict: dict, device="cuda", dtype=torch.float16):
        L.load()
        if dtype not in L.ACT_DTYPES:
            raise ValueError(f"VAE dtype must be torch.float16 or torch.bfloat16, got {dtype}")
        self.cfg = dict(cfg)
        self.dev = torch.device(device)
        self.dtype = dtype
        self.boc = list(cfg.get("block_out_channels", (128, 256, 512, 512)))
        self.lpb = cfg.get("layers_per_block", 2)
        self.latent_ch = cfg.get("latent_channels", 4)
        self.out_ch = cfg.get("out_channels", 3)
        self.groups = cfg.get("norm_num_groups", 32)
        self.scaling = cfg.get("scaling_factor", 0.18215)
        self._pack(state_dict)

    def _pack(self, sd):
        P = _Packer(sd, self.dev, self.dtype)
        w = {}

        def resnet(p):
            r = {"n1g": P.f32(p + ".norm1.weight"), "n1b": P.f32(p + ".norm1.bias"),
                 "c1": P.conv3(p + ".conv1"), "c1b": P.bias(p + ".conv1"),
                 "n2g": P.f32(p + ".norm2.weight"), "n2b": P.f32(p + ".norm2.bias"),
                 "c2": P.conv3(p + ".conv2"), "c2b": P.bias(p + ".conv2")}
            if (p + ".conv_shortcut.weight") in sd:
                r["sc"], r["scb"] = P.lin(p + ".conv_shortcut"), P.bias(p + ".conv_shortcut")
            w[p] = r

        w["pq"] = {"w": _w2d(sd, "post_quant_conv.weight").float().to(self.dev).contiguous(),
                   "b": P.f32("post_quant_conv.bias")}
        w["conv_in"] = {"w": P.conv3("decoder.conv_in", pad_in=8), "b": P.bias("decoder.conv_in")}
        resnet("decoder.mid_block.resnets.0")
        a = "decoder.mid_block.attentions.0"
        w[a] = {"ng": P.f32(a + ".group_norm.weight"), "nb": P.f32(a + ".group_norm.bias"),
                "q": P.lin(a + ".to_q"), "qb": P.bias(a + ".to_q"),
                "k": P.lin(a + ".to_k"), "kb": P.bias(a + ".to_k"),
                "v": P.lin(a + ".to_v"), "vb": P.bias(a + ".to_v"),
                "o": P.lin(a + ".to_out.0"), "ob": P.bias(a + ".to_out.0")}
        resnet("decoder.mid_block.resnets.1")
        for i in range(len(self.boc)):
            for j in range(self.lpb + 1):
                resnet(f"decoder.up_blocks.{i}.resnets.{j}")
            if i != len(self.boc) - 1:
                p = f"decoder.up_blocks.{i}.upsamplers.0.conv"
                w[p] = {"w": P.conv3(p), "b": P.bias(p)}
        w["out"] = {"g": P.f32("decoder.conv_norm_out.weight"), "b": P.f32("decoder.conv_norm_out.bias"),
                    "w": P.conv3("decoder.conv_out"), "cb": P.bias("decoder.conv_out")}
        self.w = w

    def _resnet(self, p, x):
        r = self.w[p]
        n, h, wd, _ = x.shape
        hh = L.group_norm(x, r["n1g"], r["n1b"], self.groups, 1e-6, silu=True)
        hh = L.conv3x3(hh, r["c1"], r["c1b"])
        hh = L.group_norm(hh, r["n2g"], r["n2b"], self.groups, 1e-6, silu=True)
        res = L.linear(x.reshape(n * h * wd, -1), r["sc"], r["scb"], static_w=True) if "sc" in r else x
        return L.conv3x3(hh, r["c2"], r["c2b"], res)

    def _attention(self, p, x):
        a = self.w[p]
        n, h, wd, c = x.shape
        s = h * wd
        hn = L.group_norm(x, a["ng"], a["nb"], self.groups, 1e-6, silu=False).reshape(n * s, c)
        q = L.linear(hn, a["q"], a["qb"], static_w=True)
        k = L.linear(hn, a["k"], a["kb"], static_w=True)
        xr = x.reshape(n * s, c)
        out = torch.empty_like(xr)
        for i in range(n):
            rows = slice(i * s, (i + 1) * s)
            # V^T [c, s] = W_v [c, c] . X^T : the "weight" operand is the activation matrix; the to_v bias
            # is added after P V instead (softmax rows sum to one, so P (V + 1 b^T) = P V + 1 b^T)
            vt = L.linear(a["v"], hn[rows])
            scores = L.linear(q[rows], k[rows], out_dtype=torch.float32)
            prob = L.softmax_rows(scores, c ** -0.5, out_dtype=x.dtype)
            att = L.linear(prob, vt, a["vb"])
            L.linear(att, a["o"], a["ob"], xr[rows], out=out[rows], static_w=True)
        return out.reshape(n, h, wd, c)

    def forward(self, z):
        """z: fp32 NCHW latents (unscaled, as the pipeline holds them).  Returns NHWC fp32 image
        in [-1, 1]-ish range (before the pipeline's clip)."""
        w = self.w
        x = L.latent_prep(z, w["pq"]["w"], w["pq"]["b"], 1.0, c_pad=8, out_dtype=self.dtype)
        x = L.conv3x3(x, w["conv_in"]["w"], w["conv_in"]["b"])
        x = self._resnet("decoder.mid_block.resnets.0", x)
        x = self._attention("decoder.mid_block.attentions.0", x)
        x = self._resnet("decoder.mid_block.resnets.1", x)
        for i in range(len(self.boc)):
            for j in range(self.lpb + 1):
                x = self._resnet(f"decoder.up_blocks.{i}.resnets.{j}", x)
            if i != len(self.boc) - 1:
                u = w[f"decoder.up_blocks.{i}.upsamplers.0.conv"]
                x = L.conv3x3(L.upsample2x(x), u["w"], u["b"])
        o = w["out"]
        x = L.group_norm(x, o["g"], o["b"], self.groups, 1e-6, silu=True)
        return L.conv3x3(x, o["w"], o["cb"], out_dtype=torch.float32)


class VAEDecoderModel(B200Model):
    """``vae_decoder(z) -> {"image": fp32 (B, 3, 8H, 8W)}`` (pipeline.py:313-316; z is already divided by the
    scaling factor by the caller, exactly as in the reference).  dtype=torch.bfloat16 runs the bf16 engine and
    declares z float32, as the reference declares the input of a VAE it converts in FLOAT32."""

    def __init__(self, cfg, state_dict, batch=1, height=64, width=64, device="cuda", io_dtype=np.float16,
                 dtype=torch.float16):
        self.engine = VAEDecoderEngine(cfg, state_dict, device, dtype=dtype)
        if dtype == torch.bfloat16:
            io_dtype = np.float32
        spec = {"z": {"shape": (batch, self.engine.latent_ch, height, width), "dtype": np.dtype(io_dtype)}}
        super().__init__(spec, device)
        self._z = torch.zeros(batch, self.engine.latent_ch, height, width, dtype=torch.float32, device=self.device)
        self.scale = 2 ** (len(self.engine.boc) - 1)

    def decode_device(self, z):
        """CUDA fp32 NCHW z -> NHWC fp32 image (unclipped)."""
        self._z.copy_(z)
        return self.engine.forward(self._z)

    def __call__(self, **kwargs):
        self._verify_inputs(**kwargs)
        if "z" not in kwargs:
            raise ValueError("Missing inputs: ['z']")
        as_numpy = isinstance(kwargs["z"], np.ndarray)
        self._to_device(kwargs["z"], self._z)
        img = self.engine.forward(self._z)
        nchw = L.nhwc_to_nchw_f32(img, c=self.engine.out_ch)
        return {"image": nchw.cpu().numpy() if as_numpy else nchw}


class VAEEncoderEngine(VAEDecoderEngine):
    """``quant_conv(encoder(x))`` of diffusers' AutoencoderKL (``convert_vae_encoder``, torch2coreml.py:700-796):
    the img2img entry of the Swift pipeline (Encoder.swift).  Same kernels as the decoder; the stride-2
    downsampling convolutions pad after the last row / column only (``pad_after_only``)."""

    def _pack(self, sd):
        P = _Packer(sd, self.dev, self.dtype)
        w = {}

        def resnet(p):
            r = {"n1g": P.f32(p + ".norm1.weight"), "n1b": P.f32(p + ".norm1.bias"),
                 "c1": P.conv3(p + ".conv1"), "c1b": P.bias(p + ".conv1"),
                 "n2g": P.f32(p + ".norm2.weight"), "n2b": P.f32(p + ".norm2.bias"),
                 "c2": P.conv3(p + ".conv2"), "c2b": P.bias(p + ".conv2")}
            if (p + ".conv_shortcut.weight") in sd:
                r["sc"], r["scb"] = P.lin(p + ".conv_shortcut"), P.bias(p + ".conv_shortcut")
            w[p] = r

        w["conv_in"] = {"w": P.conv3("encoder.conv_in", pad_in=8), "b": P.bias("encoder.conv_in")}
        for i in range(len(self.boc)):
            for j in range(self.lpb):
                resnet(f"encoder.down_blocks.{i}.resnets.{j}")
            if i != len(self.boc) - 1:
                p = f"encoder.down_blocks.{i}.downsamplers.0.conv"
                w[p] = {"w": P.conv3(p), "b": P.bias(p)}
        resnet("encoder.mid_block.resnets.0")
        a = "encoder.mid_block.attentions.0"
        w[a] = {"ng": P.f32(a + ".group_norm.weight"), "nb": P.f32(a + ".group_norm.bias"),
                "q": P.lin(a + ".to_q"), "qb": P.bias(a + ".to_q"),
                "k": P.lin(a + ".to_k"), "kb": P.bias(a + ".to_k"),
                "v": P.lin(a + ".to_v"), "vb": P.bias(a + ".to_v"),
                "o": P.lin(a + ".to_out.0"), "ob": P.bias(a + ".to_out.0")}
        resnet("encoder.mid_block.resnets.1")
        # conv_out (2 * latent moments) followed by the 1x1 quant_conv: folded into one 3x3 convolution,
        # W' = Wq . Wc per tap, b' = Wq bc + bq (both are linear maps with nothing in between)
        wq = _w2d(sd, "quant_conv.weight").float()
        wc = sd["encoder.conv_out.weight"].float()
        wf = torch.einsum("om,mikl->oikl", wq, wc)
        bf = wq @ sd["encoder.conv_out.bias"].float() + sd["quant_conv.bias"].float()
        w["out"] = {"g": P.f32("encoder.conv_norm_out.weight"), "b": P.f32("encoder.conv_norm_out.bias"),
                    "w": P.f16(wf.permute(0, 2, 3, 1).reshape(wf.shape[0], -1)),
                    "cb": bf.to(device=self.dev, dtype=torch.float32).contiguous()}
        self.moments = wf.shape[0]
        self.w = w

    def forward(self, x):
        """x: fp32 / fp16 NCHW image in [-1, 1].  Returns NHWC fp32 moments [B, H/8, W/8, 2 * latent]."""
        w = self.w
        h = L.conv3x3(L.nchw_to_nhwc(x, c_pad=8, out_dtype=self.dtype), w["conv_in"]["w"], w["conv_in"]["b"])
        for i in range(len(self.boc)):
            for j in range(self.lpb):
                h = self._resnet(f"encoder.down_blocks.{i}.resnets.{j}", h)
            if i != len(self.boc) - 1:
                d = w[f"encoder.down_blocks.{i}.downsamplers.0.conv"]
                h = L.conv3x3(h, d["w"], d["b"], stride=2, pad_after_only=True)
        h = self._resnet("encoder.mid_block.resnets.0", h)
        h = self._attention("encoder.mid_block.attentions.0", h)
        h = self._resnet("encoder.mid_block.resnets.1", h)
        o = w["out"]
        h = L.group_norm(h, o["g"], o["b"], self.groups, 1e-6, silu=True)
        return L.conv3x3(h, o["w"], o["cb"], out_dtype=torch.float32)


class VAEEncoderModel(B200Model):
    """``vae_encoder(x) -> {"latent": fp32 (B, 2 * latent_channels, H/8, W/8)}`` (torch2coreml.py:751-756: the
    moments; sampling and scaling happen in the caller, Encoder.swift).  dtype=torch.bfloat16 runs the bf16 engine
    and declares x float32."""

    def __init__(self, cfg, state_dict, batch=1, height=512, width=512, device="cuda", io_dtype=np.float16,
                 dtype=torch.float16):
        self.engine = VAEEncoderEngine(cfg, state_dict, device, dtype=dtype)
        if dtype == torch.bfloat16:
            io_dtype = np.float32
        spec = {"x": {"shape": (batch, 3, height, width), "dtype": np.dtype(io_dtype)}}
        super().__init__(spec, device)
        self._x = torch.zeros(batch, 3, height, width, dtype=torch.float32, device=self.device)

    def __call__(self, **kwargs):
        self._verify_inputs(**kwargs)
        if "x" not in kwargs:
            raise ValueError("Missing inputs: ['x']")
        as_numpy = isinstance(kwargs["x"], np.ndarray)
        self._to_device(kwargs["x"], self._x)
        mom = self.engine.forward(self._x)
        nchw = L.nhwc_to_nchw_f32(mom, c=self.engine.moments)
        return {"latent": nchw.cpu().numpy() if as_numpy else nchw}

    def encode(self, x, noise, scaling_factor=None):
        """Swift Encoder.encode: latent = (mean + exp(0.5 * clamp(logvar, -30, 20)) * noise) * scaling_factor."""
        mom = self(x=x)["latent"]
        mom = torch.as_tensor(mom)
        mean, logvar = mom.chunk(2, dim=1)
        sf = self.engine.scaling if scaling_factor is None else scaling_factor
        return (mean + torch.exp(0.5 * logvar.clamp(-30.0, 20.0)) * torch.as_tensor(noise).to(mean)) * sf
