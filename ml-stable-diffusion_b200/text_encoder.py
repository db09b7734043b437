"""CLIP text encoder on the sm_90a kernels (SURVEY 8f N2, device half).

Replaces the ``text_encoder`` Core ML model of the reference -- ``transformers.CLIPTextModel`` as converted by
``torch2coreml.py:408-441`` and called by ``pipeline.py:151-175`` with *float* ``input_ids`` (1, 77), returning
``last_hidden_state`` (1, 77, D).  Pre-LayerNorm transformer: x += out_proj(causal_attention(LN1(x)));
x += fc2(act(fc1(LN2(x)))); final LayerNorm.  q/k/v are one fused GEMM, the causal softmax runs in the flash
attention kernel (d_head = 64 for both CLIP-L and OpenCLIP-H), GELU / quick-GELU in the GEMM epilogue.
"""
from __future__ import annotations

import numpy as np
import torch

from . import lib as L
from .model import B200Model

_ACT = {"gelu": 2, "quick_gelu": 3}


class TextEncoderEngine:
    def __init__(self, cfg: dict, state_dict: dict, device="cuda"):
        L.load()
        self.cfg = dict(cfg)
        self.dev = torch.device(device)
        self.d = cfg["hidden_size"]
        self.heads = cfg["num_attention_heads"]
        if self.d // self.heads != 64:
            raise L.B200SDError(f"text encoder head dim {self.d // self.heads} not supported by the attention kernel (64)")
        if cfg["hidden_act"] not in _ACT:
            raise L.B200SDError(f"unsupported hidden_act {cfg['hidden_act']!r}")
        self.act = _ACT[cfg["hidden_act"]]
        self.eps = cfg.get("layer_norm_eps", 1e-5)
        self.layers = cfg["num_hidden_layers"]
        self.seq = cfg["max_position_embeddings"]
        self._pack(state_dict)

    def _pack(self, sd):
        dev = self.dev

        def f16(k):
            return sd[k].detach().to(device=dev, dtype=torch.float16).contiguous()

        def f32(k):
            return sd[k].detach().to(device=dev, dtype=torch.float32).contiguous()

        self.proj = None
        if "text_projection.weight" in sd:  # CLIPTextModelWithProjection (SDXL's second encoder)
            self.proj = f16("text_projection.weight")
        w = {"tok": f16("text_model.embeddings.token_embedding.weight"),
             "pos": f16("text_model.embeddings.position_embedding.weight"),
             "lnf_g": f32("text_model.final_layer_norm.weight"), "lnf_b": f32("text_model.final_layer_norm.bias"),
             "layers": []}
        for i in range(self.layers):
            p = f"text_model.encoder.layers.{i}."
            qkv = torch.cat([sd[p + f"self_attn.{n}.weight"].detach().float() for n in ("q_proj", "k_proj", "v_proj")], 0)
            qkv_b = torch.cat([sd[p + f"self_attn.{n}.bias"].detach().float() for n in ("q_proj", "k_proj", "v_proj")], 0)
            w["layers"].append({
                "ln1_g": f32(p + "layer_norm1.weight"), "ln1_b": f32(p + "layer_norm1.bias"),
                "qkv": qkv.to(device=dev, dtype=torch.float16).contiguous(), "qkv_b": qkv_b.to(dev).contiguous(),
                "o": f16(p + "self_attn.out_proj.weight"), "o_b": f32(p + "self_attn.out_proj.bias"),
                "ln2_g": f32(p + "layer_norm2.weight"), "ln2_b": f32(p + "layer_norm2.bias"),
                "fc1": f16(p + "mlp.fc1.weight"), "fc1_b": f32(p + "mlp.fc1.bias"),
                "fc2": f16(p + "mlp.fc2.weight"), "fc2_b": f32(p + "mlp.fc2.bias"),
            })
        self.w = w

    def forward(self, ids, hidden_layer=None):
        """ids: CUDA fp32 [B, S] -> (last_hidden_state fp16 [B*S, D] after the final LayerNorm,
        hidden_states[hidden_layer] fp16 [B*S, D] or None).  hidden_states follows transformers: entry 0 is the
        embedding output, entry i the output of layer i (before the final LayerNorm); SDXL uses -2
        (torch2coreml.py:431-433)."""
        w, d = self.w, self.d
        b, s = ids.shape
        want = None if hidden_layer is None else hidden_layer % (self.layers + 1)
        x = L.embed_tokens(ids, w["tok"], w["pos"])
        picked = x if want == 0 else None
        for i, ly in enumerate(w["layers"]):
            n1 = L.layer_norm(x, ly["ln1_g"], ly["ln1_b"], eps=self.eps)
            qkv = L.linear(n1, ly["qkv"], ly["qkv_b"], static_w=True)
            a = L.attention(qkv[:, :d], qkv[:, d:2 * d], qkv[:, 2 * d:], b, self.heads, s, s, causal=True)
            x = L.linear(a, ly["o"], ly["o_b"], x, static_w=True)
            n2 = L.layer_norm(x, ly["ln2_g"], ly["ln2_b"], eps=self.eps)
            hdn = L.linear(n2, ly["fc1"], ly["fc1_b"], act=self.act, static_w=True)
            x = L.linear(hdn, ly["fc2"], ly["fc2_b"], x, static_w=True)
            if want == i + 1:
                picked = x
        return L.layer_norm(x, w["lnf_g"], w["lnf_b"], eps=self.eps), picked

    def pooled(self, last_hidden, eos_rows):
        """last_hidden fp16 [B*S, D]; eos_rows: LongTensor of the flattened end-of-text row per batch element ->
        pooler_output, or text_embeds = text_projection(pooler_output) when the checkpoint has a projection."""
        pooled = last_hidden.index_select(0, eos_rows).float().contiguous()
        if self.proj is None:
            return pooled
        return L.linear_small(pooled, self.proj)  # [B, D] x [P, D]^T: weight-bandwidth bound, fp32 accumulate


class TextEncoderModel(B200Model):
    """``text_encoder(input_ids=float32 (B, 77))`` (pipeline.py:170-175; the reference passes the ids as float32).
    Outputs follow torch2coreml.py:443-446: ``last_hidden_state`` + ``pooled_outputs``, or for SDXL
    (``hidden_layer=-2``) ``hidden_embeds`` + ``pooled_outputs`` (the second encoder's pooled output is its
    ``text_embeds``)."""

    def __init__(self, cfg, state_dict, batch=1, device="cuda", hidden_layer=None):
        self.engine = TextEncoderEngine(cfg, state_dict, device)
        self.batch, self.seq, self.hidden = batch, self.engine.seq, self.engine.d
        self.hidden_layer = hidden_layer
        self.eos_token_id = cfg.get("eos_token_id", cfg["vocab_size"] - 1)
        spec = {"input_ids": {"shape": (batch, self.seq), "dtype": np.dtype(np.float32)}}
        super().__init__(spec, device)
        self._ids = torch.zeros(batch, self.seq, dtype=torch.float32, device=self.device)

    def _eos_rows(self):
        ids = self._ids.long()
        hit = ids == self.eos_token_id
        pos = torch.where(hit.any(-1), hit.int().argmax(-1), ids.argmax(-1))  # modeling_clip.py pooling rule
        return pos + torch.arange(self.batch, device=self.device) * self.seq

    def __call__(self, **kwargs):
        self._verify_inputs(**kwargs)
        if "input_ids" not in kwargs:
            raise ValueError("Missing inputs: ['input_ids']")
        as_numpy = isinstance(kwargs["input_ids"], np.ndarray)
        self._to_device(kwargs["input_ids"], self._ids)
        last, picked = self.engine.forward(self._ids, self.hidden_layer)
        pooled = self.engine.pooled(last, self._eos_rows()).float()
        if self.hidden_layer is None:
            out = {"last_hidden_state": last.float().reshape(self.batch, self.seq, self.hidden), "pooled_outputs": pooled}
        else:
            out = {"hidden_embeds": picked.float().reshape(self.batch, self.seq, self.hidden), "pooled_outputs": pooled}
        return {k: v.cpu().numpy() for k, v in out.items()} if as_numpy else out
