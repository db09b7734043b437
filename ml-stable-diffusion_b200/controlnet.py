"""ControlNet on the sm_90a kernels: the UNet encoder half + mid block + 1x1 "zero convs" and the
8-conv conditioning embedder (reference ``python_coreml_stable_diffusion/controlnet.py:15-250``), with the
reference's model-call contract (``pipeline.py:259-284``: ``sample, timestep, encoder_hidden_states,
controlnet_cond`` -> ``additional_residual_i``).  Re-uses ``UNetEngine``'s packed blocks; the conditioning
embedder's SiLU is fused into the conv epilogue (``act=1``)."""
from __future__ import annotations

import numpy as np
import torch

from . import lib as L
from .model import B200Model
from .unet import UNetEngine, _Packer


class ControlNetEngine(UNetEngine):
    def __init__(self, cfg: dict, state_dict: dict, device="cuda"):
        cfg = dict(cfg)
        # the encoder half is built by the UNet packer: give it no up path and no output head
        self._ce_channels = list(cfg.get("conditioning_embedding_out_channels", (16, 32, 96, 256)))
        self._full_sd = state_dict
        # mid block transformer depth is 1 regardless of transformer_layers_per_block (controlnet.py:168-180)
        ucfg = dict(cfg, up_block_types=(), out_channels=cfg.get("in_channels", 4), mid_block_transformer_layers=1)
        super().__init__(ucfg, state_dict, device)

    def _pack(self, sd):
        # reuse the UNet packer for conv_in / time / down / mid; skip what a ControlNet does not have
        shim = dict(sd)
        for k in ("conv_norm_out.weight", "conv_norm_out.bias"):
            shim.setdefault(k, torch.ones(self.boc[0]))
        shim.setdefault("conv_out.weight", torch.zeros(self.out_ch, self.boc[0], 3, 3))
        shim.setdefault("conv_out.bias", torch.zeros(self.out_ch))
        super()._pack(shim)
        P = _Packer(sd, self.dev)
        ce = self._ce_channels
        emb = [{"w": P.conv3("controlnet_cond_embedding.conv_in", pad_in=8),
                "b": P.bias("controlnet_cond_embedding.conv_in"), "stride": 1, "act": 1}]
        for i in range(len(ce) - 1):
            for j, st in ((2 * i, 1), (2 * i + 1, 2)):
                n = f"controlnet_cond_embedding.blocks.{j}"
                emb.append({"w": P.conv3(n), "b": P.bias(n), "stride": st, "act": 1})
        emb.append({"w": P.conv3("controlnet_cond_embedding.conv_out"),
                    "b": P.bias("controlnet_cond_embedding.conv_out"), "stride": 1, "act": 0})
        self.embedder = emb
        self.zero_convs = []
        k = 0
        while f"controlnet_down_blocks.{k}.weight" in sd:
            n = f"controlnet_down_blocks.{k}"
            self.zero_convs.append((P.lin(n), P.bias(n)))
            k += 1
        self.zero_mid = (P.lin("controlnet_mid_block"), P.bias("controlnet_mid_block"))

    def embed_condition(self, cond_nhwc):
        """controlnet_cond (NHWC fp16, 3 channels padded to 8) -> (B, H/8, W/8, C0) embedding.  The hint image
        is the same for every denoising step, so callers may compute this once per image (the reference
        recomputes it every step, pipeline.py:516-522)."""
        x = cond_nhwc
        for e in self.embedder:
            x = L.conv3x3(x, e["w"], e["b"], stride=e["stride"], act=e["act"])
        return x

    def forward(self, sample, timesteps, ctx_tokens, s_ctx, cond_nhwc, temb_all=None, kv_all=None, emb=None):
        """Returns the list of NHWC fp16 residuals: 12 (or fewer) down residuals + the mid residual.
        temb_all / kv_all / emb: precomputed time-embedding biases, cross-attention K/V and conditioning embedding
        (constant over a denoising loop: the pipeline's per-prompt prologue)."""
        batch = sample.shape[0]
        if temb_all is None:
            temb_all = self.time_embedding(timesteps)
        if kv_all is None:
            kv_all = self.kv_project(ctx_tokens)
        e = self.embed_condition(cond_nhwc) if emb is None else emb
        if self.fused:
            st = {}
            x = L.conv3x3(sample, self.w["conv_in"]["w"], self.w["conv_in"]["b"], e, stats=st if self.fuse_gn else None)
            xs = st.get("chan")
            skips = [x]
            for i, typ in enumerate(self.down_types):
                for j in range(self.lpb):
                    x, xs = self._resnet_f(f"down_blocks.{i}.resnets.{j}", x, xs, None, None, temb_all)
                    if typ == "CrossAttnDownBlock2D":
                        x, xs = self._transformer_f(f"down_blocks.{i}.attentions.{j}", x, xs, kv_all, batch, self.heads[i], s_ctx)
                    skips.append(x)
                if i != self.nb - 1:
                    d = self.w[f"down_blocks.{i}.downsamplers.0.conv"]
                    st = {}
                    x = L.conv3x3(x, d["w"], d["b"], stride=2, stats=st if self.fuse_gn else None)
                    xs = st.get("chan")
                    skips.append(x)
            x, xs = self._resnet_f("mid_block.resnets.0", x, xs, None, None, temb_all)
            x, xs = self._transformer_f("mid_block.attentions.0", x, xs, kv_all, batch, self.heads[-1], s_ctx)
            x, xs = self._resnet_f("mid_block.resnets.1", x, xs, None, None, temb_all)
        else:
            x = L.conv3x3(sample, self.w["conv_in"]["w"], self.w["conv_in"]["b"], e)   # conv_in(sample) + embedding
            skips = [x]
            for i, typ in enumerate(self.down_types):
                for j in range(self.lpb):
                    x = self._resnet(f"down_blocks.{i}.resnets.{j}", x, None, temb_all)
                    if typ == "CrossAttnDownBlock2D":
                        x = self._transformer(f"down_blocks.{i}.attentions.{j}", x, kv_all, batch, self.heads[i], s_ctx)
                    skips.append(x)
                if i != self.nb - 1:
                    d = self.w[f"down_blocks.{i}.downsamplers.0.conv"]
                    x = L.conv3x3(x, d["w"], d["b"], stride=2)
                    skips.append(x)
            x = self._resnet("mid_block.resnets.0", x, None, temb_all)
            x = self._transformer("mid_block.attentions.0", x, kv_all, batch, self.heads[-1], s_ctx)
            x = self._resnet("mid_block.resnets.1", x, None, temb_all)
        outs = []
        for s, (w, b) in zip(skips, self.zero_convs):
            n, h, wd, c = s.shape
            outs.append(L.linear(s.reshape(n * h * wd, c), w, b, static_w=True).reshape(n, h, wd, c))
        n, h, wd, c = x.shape
        outs.append(L.linear(x.reshape(n * h * wd, c), self.zero_mid[0], self.zero_mid[1], static_w=True).reshape(n, h, wd, c))
        return outs


class ControlNetModel(B200Model):
    """``controlnet(sample, timestep, encoder_hidden_states, controlnet_cond) -> {"additional_residual_i": ...}``
    (pipeline.py:259-284, torch2coreml.py:1382-1412)."""

    def __init__(self, cfg, state_dict, batch=2, height=64, width=64, seq_len=77, device="cuda", io_dtype=np.float16,
                 use_cuda_graph=True):
        self.engine = ControlNetEngine(cfg, state_dict, device)
        self.use_cuda_graph = use_cuda_graph
        self._graph = None
        self._outs = None
        e = self.engine
        self.batch, self.h, self.w, self.seq = batch, height, width, seq_len
        dt = np.dtype(io_dtype)
        spec = {
            "sample": {"shape": (batch, e.in_ch, height, width), "dtype": dt},
            "timestep": {"shape": (batch,), "dtype": dt},
            "encoder_hidden_states": {"shape": (batch, cfg["cross_attention_dim"], 1, seq_len), "dtype": dt},
            "controlnet_cond": {"shape": (batch, 3, height * 8, width * 8), "dtype": dt},
        }
        super().__init__(spec, device)
        dev = self.device
        self._sample = torch.zeros(spec["sample"]["shape"], dtype=torch.float32, device=dev)
        self._t = torch.zeros(batch, dtype=torch.float32, device=dev)
        self._ctx = torch.zeros(spec["encoder_hidden_states"]["shape"], dtype=torch.float16, device=dev)
        self._cond = torch.zeros(spec["controlnet_cond"]["shape"], dtype=torch.float16, device=dev)
        self._kv_all = (torch.zeros(batch * seq_len, e.kv_total, dtype=torch.float16, device=dev)
                        if e.kv_w is not None else None)
        self._emb = None     # conditioning embedding of `_cond` (device loop prologue)
        self._table = None   # time-embedding biases of all steps (device loop prologue)

    # -- per-prompt prologue + per-step core of the device loop (pipeline.denoise) ------------------------------
    def prepare_prompt(self, ts_rows):
        """Everything that does not change over a denoising loop: cross-attention K/V from `_ctx`, the embedding of
        the conditioning image `_cond` (the reference recomputes it every step, pipeline.py:516-522), the
        time-embedding biases of all steps."""
        e, b = self.engine, self.batch
        if self._kv_all is not None:
            e.kv_project(L.ctx_to_tokens(self._ctx), out=self._kv_all)
        self._emb = e.embed_condition(L.nchw_to_nhwc(self._cond, c_pad=8))
        n_steps = ts_rows.shape[0] // b
        per = max(1, 32 // b)
        parts = [e.time_embedding(ts_rows[s0 * b:(s0 + min(per, n_steps - s0)) * b].contiguous())
                 for s0 in range(0, n_steps, per)]
        self._table = torch.cat(parts, 0).reshape(n_steps, b, -1)

    def run_core(self, x_nhwc, step):
        """Residuals (NHWC fp16) for the UNet input `x_nhwc` at loop step `step` (after prepare_prompt)."""
        return self.engine.forward(x_nhwc, None, None, self.seq, None, temb_all=self._table[step], kv_all=self._kv_all,
                                   emb=self._emb)

    def _run(self):
        e = self.engine
        x = L.nchw_to_nhwc(self._sample, c_pad=e.in_pad)
        ctx = L.ctx_to_tokens(self._ctx)
        cond = L.nchw_to_nhwc(self._cond, c_pad=8)
        return e.forward(x, self._t, ctx, self.seq, cond)

    def forward_device(self):
        """Static input buffers -> list of NHWC fp16 residuals.  With CUDA graphs the list is a set of static
        tensors owned by the captured graph (overwritten by the next call)."""
        if not self.use_cuda_graph:
            return self._run()
        if self._graph is None:
            s = torch.cuda.Stream(device=self.device)  # warm-up outside capture: workspace / weight tiling
            s.wait_stream(torch.cuda.current_stream())
            with torch.cuda.stream(s):
                self._run()
            torch.cuda.current_stream().wait_stream(s)
            torch.cuda.synchronize()
            g = torch.cuda.CUDAGraph()
            with torch.cuda.graph(g):
                self._outs = self._run()
            self._graph = g
        self._graph.replay()
        return self._outs

    def __call__(self, **kwargs):
        self._verify_inputs(**kwargs)
        missing = [k for k in self.expected_inputs if k not in kwargs]
        if missing:
            raise ValueError(f"Missing inputs: {missing}")
        as_numpy = isinstance(kwargs["sample"], np.ndarray)
        self._to_device(kwargs["sample"], self._sample)
        self._to_device(kwargs["timestep"], self._t)
        self._to_device(kwargs["encoder_hidden_states"], self._ctx)
        self._to_device(kwargs["controlnet_cond"], self._cond)
        outs = self.forward_device()
        res = {}
        for i, o in enumerate(outs):
            nchw = L.nhwc_to_nchw_f32(o)
            res[f"additional_residual_{i}"] = nchw.cpu().numpy() if as_numpy else nchw
        return res
