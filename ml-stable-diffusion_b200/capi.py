"""ctypes binding of the model-level C-ABI (``b200sd_unet_create / _prepare_prompt / _forward / b200sd_destroy``,
include/b200sd.h): what a non-Python host (the reference's Swift front end, ``Unet.swift:90-144``) would call.  The
handle owns packed weights, activation arena and launch sequence; this wrapper only converts a diffusers-style config
and state dict into the C structs and passes DEVICE pointers per call.  Used by the parity tests and as the worked
example in INTEGRATION.md; the Python pipeline itself drives the same kernels through ``unet.UNetEngine``."""
from __future__ import annotations

import ctypes as C

import torch

from . import lib as L


class UNetConfig(C.Structure):
    _fields_ = [
        ("in_channels", C.c_int32), ("out_channels", C.c_int32), ("layers_per_block", C.c_int32),
        ("norm_num_groups", C.c_int32), ("cross_attention_dim", C.c_int32), ("norm_eps", C.c_float),
        ("n_blocks", C.c_int32), ("block_out_channels", C.c_int32 * 8), ("attention_heads", C.c_int32 * 8),
        ("transformer_layers", C.c_int32 * 8), ("mid_transformer_layers", C.c_int32), ("down_cross_attn", C.c_int32 * 8),
        ("up_cross_attn", C.c_int32 * 8), ("flip_sin_to_cos", C.c_int32), ("freq_shift", C.c_float),
        ("addition_embed_text_time", C.c_int32), ("addition_time_embed_dim", C.c_int32),
        ("projection_class_embeddings_input_dim", C.c_int32), ("num_time_ids", C.c_int32),
        ("support_controlnet", C.c_int32), ("batch", C.c_int32), ("height", C.c_int32), ("width", C.c_int32),
        ("seq_len", C.c_int32),
    ]


class Weight(C.Structure):
    _fields_ = [("name", C.c_char_p), ("data", C.c_void_p), ("dtype", C.c_int32), ("ndim", C.c_int32),
                ("shape", C.c_int64 * 4)]


def _as_list(v, n):
    return list(v) if isinstance(v, (list, tuple)) else [v] * n


def make_config(cfg: dict, batch: int, height: int, width: int, seq_len: int = 77) -> UNetConfig:
    """The reference's UNet config keys (unet.py:733-800) -> ``b200sd_unet_config``."""
    if cfg.get("time_cond_proj_dim"):
        raise ValueError(f"the C handle takes no time condition: a UNet with time_cond_proj_dim="
                         f"{cfg['time_cond_proj_dim']} (guidance embedding) runs through UNetModel only")
    boc = list(cfg["block_out_channels"])
    nb = len(boc)
    c = UNetConfig()
    c.in_channels, c.out_channels = cfg.get("in_channels", 4), cfg.get("out_channels", 4)
    c.layers_per_block, c.norm_num_groups = cfg.get("layers_per_block", 2), cfg.get("norm_num_groups", 32)
    c.cross_attention_dim, c.norm_eps, c.n_blocks = cfg["cross_attention_dim"], cfg.get("norm_eps", 1e-5), nb
    depth = _as_list(cfg.get("transformer_layers_per_block", 1), nb)
    for i in range(nb):
        c.block_out_channels[i] = boc[i]
        c.attention_heads[i] = _as_list(cfg.get("attention_head_dim", 8), nb)[i]
        c.transformer_layers[i] = depth[i]
        c.down_cross_attn[i] = int(cfg["down_block_types"][i] == "CrossAttnDownBlock2D")
        c.up_cross_attn[i] = int(cfg["up_block_types"][i] == "CrossAttnUpBlock2D")
    c.mid_transformer_layers = cfg.get("mid_block_transformer_layers", depth[-1])
    c.flip_sin_to_cos, c.freq_shift = int(cfg.get("flip_sin_to_cos", True)), float(cfg.get("freq_shift", 0))
    c.addition_embed_text_time = int(cfg.get("addition_embed_type") == "text_time")
    c.addition_time_embed_dim = cfg.get("addition_time_embed_dim", 0) or 0
    c.projection_class_embeddings_input_dim = cfg.get("projection_class_embeddings_input_dim", 0) or 0
    c.num_time_ids = cfg.get("num_time_ids", 6)
    c.support_controlnet = int(bool(cfg.get("support_controlnet", False)))
    c.batch, c.height, c.width, c.seq_len = batch, height, width, seq_len
    return c


class CUNet:
    """Opaque-handle UNet.  All call arguments are CUDA tensors; only their device pointers cross the boundary."""

    def __init__(self, cfg: dict, state_dict: dict, batch=2, height=64, width=64, seq_len=77):
        lib = L.load()
        self.cfg = make_config(cfg, batch, height, width, seq_len)
        keep, arr = [], (Weight * len(state_dict))()
        for i, (k, v) in enumerate(state_dict.items()):
            t = v.detach().cpu().contiguous()
            if t.dtype not in (torch.float16, torch.float32):
                t = t.float()
            keep.append(t)
            arr[i].name = k.encode()
            arr[i].data = t.data_ptr()
            arr[i].dtype = 0 if t.dtype == torch.float16 else 1
            arr[i].ndim = t.dim()
            for d, sdim in enumerate(t.shape):
                arr[i].shape[d] = sdim
        self._h = C.c_void_p()
        L._check(lib.b200sd_unet_create(C.byref(self.cfg), arr, len(state_dict), L._stream(), C.byref(self._h)),
                 "b200sd_unet_create")
        self.out_shape = (batch, self.cfg.out_channels, height, width)

    def prepare_prompt(self, encoder_hidden_states):
        L._check(L.load().b200sd_unet_prepare_prompt(self._h, L._ptr(encoder_hidden_states), L._stream()),
                 "b200sd_unet_prepare_prompt")

    def forward(self, sample, timesteps, encoder_hidden_states=None, time_ids=None, text_embeds=None, residuals=None):
        out = torch.empty(self.out_shape, dtype=torch.float32, device=sample.device)
        res = None
        if residuals is not None:
            res = (C.c_void_p * len(residuals))(*[r.data_ptr() for r in residuals])
        L._check(L.load().b200sd_unet_forward(self._h, L._ptr(sample), int(sample.dtype == torch.float32), L._ptr(timesteps),
                                              L._ptr(encoder_hidden_states), L._ptr(time_ids), L._ptr(text_embeds), res,
                                              L._ptr(out), L._stream()), "b200sd_unet_forward")
        return out

    def set_attention_impl(self, impl: int):
        L._check(L.load().b200sd_unet_set_attention_impl(self._h, int(impl)), "b200sd_unet_set_attention_impl")

    def device_bytes(self) -> int:
        return int(L.load().b200sd_unet_device_bytes(self._h))

    def close(self):
        if self._h:
            L.load().b200sd_destroy(self._h)
            self._h = C.c_void_p()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass
