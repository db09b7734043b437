"""The CLIP transformer encoder both CLIP towers run: the text encoder (causal) and the safety checker's vision tower.

Pre-LayerNorm layers (transformers' ``CLIPEncoderLayer``): x += out_proj(attention(LN1(x))); x += fc2(act(fc1(LN2(x)))).
q / k / v are one fused GEMM, attention is the flash-attention kernel at d_head = 64, GELU / quick-GELU runs in the fc1
GEMM's epilogue and both residual adds in the out_proj / fc2 epilogues.
"""
from __future__ import annotations

import torch

from . import lib as L

ACT = {"gelu": 2, "quick_gelu": 3}


def pack_layers(sd, prefix, n_layers, device):
    """Device weights of ``<prefix>{i}.*`` (``text_model.encoder.layers.`` / ``vision_model.encoder.layers.``):
    fp16 GEMM weights with q / k / v concatenated, fp32 biases and LayerNorm affines."""
    def f16(k):
        return sd[k].detach().to(device=device, dtype=torch.float16).contiguous()

    def f32(k):
        return sd[k].detach().to(device=device, dtype=torch.float32).contiguous()

    layers = []
    for i in range(n_layers):
        p = f"{prefix}{i}."
        qkv = torch.cat([sd[p + f"self_attn.{n}.weight"].detach().float() for n in ("q_proj", "k_proj", "v_proj")], 0)
        qkv_b = torch.cat([sd[p + f"self_attn.{n}.bias"].detach().float() for n in ("q_proj", "k_proj", "v_proj")], 0)
        layers.append({
            "ln1_g": f32(p + "layer_norm1.weight"), "ln1_b": f32(p + "layer_norm1.bias"),
            "qkv": qkv.to(device=device, dtype=torch.float16).contiguous(), "qkv_b": qkv_b.to(device).contiguous(),
            "o": f16(p + "self_attn.out_proj.weight"), "o_b": f32(p + "self_attn.out_proj.bias"),
            "ln2_g": f32(p + "layer_norm2.weight"), "ln2_b": f32(p + "layer_norm2.bias"),
            "fc1": f16(p + "mlp.fc1.weight"), "fc1_b": f32(p + "mlp.fc1.bias"),
            "fc2": f16(p + "mlp.fc2.weight"), "fc2_b": f32(p + "mlp.fc2.bias"),
        })
    return layers


def run_layers(x, layers, batch, seq, d, heads, act, eps, causal, on_layer=None):
    """x fp16 [batch * seq, d] through every layer; ``on_layer(i, x)`` sees the output of layer i.  Returns the last
    layer's output."""
    for i, ly in enumerate(layers):
        n1 = L.layer_norm(x, ly["ln1_g"], ly["ln1_b"], eps=eps)
        qkv = L.linear(n1, ly["qkv"], ly["qkv_b"], static_w=True)
        a = L.attention(qkv[:, :d], qkv[:, d:2 * d], qkv[:, 2 * d:], batch, heads, seq, seq, causal=causal)
        x = L.linear(a, ly["o"], ly["o_b"], x, static_w=True)
        n2 = L.layer_norm(x, ly["ln2_g"], ly["ln2_b"], eps=eps)
        hdn = L.linear(n2, ly["fc1"], ly["fc1_b"], act=act, static_w=True)
        x = L.linear(hdn, ly["fc2"], ly["fc2_b"], x, static_w=True)
        if on_layer is not None:
            on_layer(i, x)
    return x
