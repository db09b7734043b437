"""Model-call boundary: drop-in for ``python_coreml_stable_diffusion.coreml_model.CoreMLModel``.

The reference pipeline talks to its device runtime exclusively through
``CoreMLModel(model_path, compute_unit)`` objects exposing ``expected_inputs`` (name -> shape,
dtype) and ``__call__(**np.ndarray) -> dict[str, np.ndarray]`` with strict validation
(``coreml_model.py:36-120``; tensor names/dtypes ``pipeline.py:531-536``, ``torch2coreml.py:857-863``).
``B200Model`` keeps that contract -- same names, shapes, dtypes, ``TypeError``/``ValueError``
behaviour -- and additionally accepts CUDA tensors (no host round trip; used by the pipeline's
device-resident loop).  Weights live on the GPU; the launch sequence is captured once into a CUDA
graph and replayed per call.
"""
from __future__ import annotations

import numpy as np
import torch

from . import config as C
from . import lib as L
from .unet import UNetEngine


class B200Model:
    """Base: named-tensor validation identical to ``CoreMLModel._verify_inputs`` (coreml_model.py:97-116)."""

    def __init__(self, expected_inputs, device):
        self.expected_inputs = expected_inputs
        self.device = torch.device(device)

    def _verify_inputs(self, **kwargs):
        for k, v in kwargs.items():
            if k not in self.expected_inputs:
                raise ValueError(f"Received unexpected input kwarg: {k}")
            spec = self.expected_inputs[k]
            if isinstance(v, np.ndarray):
                dt = v.dtype
            elif torch.is_tensor(v):
                dt = np.dtype(str(v.dtype).replace("torch.", ""))
            else:
                raise TypeError(f"Expected numpy.ndarray, got {v} for input: {k}")
            if not dt == spec["dtype"]:
                raise TypeError(f"Expected dtype {spec['dtype']}, got {dt} for input: {k}")
            if not tuple(v.shape) == tuple(spec["shape"]):
                raise TypeError(f"Expected shape {spec['shape']}, got {tuple(v.shape)} for input: {k}")

    def _to_device(self, v, buf):
        """Copy a numpy array / tensor into the static device buffer ``buf`` (dtype-converting)."""
        if isinstance(v, np.ndarray):
            v = torch.from_numpy(v)
        buf.copy_(v, non_blocking=True)
        return buf


class UNetModel(B200Model):
    """``unet(sample, timestep, encoder_hidden_states[, time_ids, text_embeds][, timestep_cond][,
    additional_residual_i]) -> {"noise_pred": fp32}`` (pipeline.py:531-536).  ``timestep_cond`` ([batch,
    time_cond_proj_dim], the guidance embedding): guidance-embedding (LCM) UNets only.

    The device-loop methods (``time_table``, ``prepare_prompt``, ``_run_core``, ``forward_device``) take ``rows``: run
    on the first ``rows`` images of the static buffers only (the guidance-free loop runs batch // 2 of them)."""

    def __init__(self, cfg, state_dict, batch=2, height=64, width=64, seq_len=77, device="cuda",
                 use_cuda_graph=True, io_dtype=np.float16, quantization=None, palettization=None):
        """quantization: a W8A8Recipe or the path of a saved one; palettization: n-bit palettized weights (UNetEngine)."""
        C.check_latent_size(cfg, height, width)
        self.engine = UNetEngine(cfg, state_dict, device, quantization=quantization, palettization=palettization)
        e = self.engine
        self.batch, self.h, self.w, self.seq = batch, height, width, seq_len
        self.in_channels = e.in_ch  # the reference pipeline sets/reads this (pipeline.py:104)
        dt = np.dtype(io_dtype)
        d_ctx = cfg["cross_attention_dim"]
        spec = {
            "sample": {"shape": (batch, e.in_ch, height, width), "dtype": dt},
            "timestep": {"shape": (batch,), "dtype": dt},
            "encoder_hidden_states": {"shape": (batch, d_ctx, 1, seq_len), "dtype": dt},
        }
        if e.xl:
            # SDXL base: six geometry scalars (original size, crop, target size); the refiner: five (aesthetic score in
            # place of the target size, StableDiffusionXLPipeline.swift:327-345) -> cfg["num_time_ids"] = 5
            nid = int(cfg.get("num_time_ids", 6))
            spec["time_ids"] = {"shape": (batch, nid), "dtype": dt}
            spec["text_embeds"] = {"shape": (batch, cfg["projection_class_embeddings_input_dim"]
                                             - nid * cfg["addition_time_embed_dim"]), "dtype": dt}
        if e.time_cond_dim:
            spec["timestep_cond"] = {"shape": (batch, e.time_cond_dim), "dtype": dt}
        self.res_shapes = []
        if e.support_controlnet:
            for i, shp in enumerate(self.residual_shapes()):
                spec[f"additional_residual_{i}"] = {"shape": shp, "dtype": dt}
                self.res_shapes.append(shp)
        super().__init__(spec, device)
        dev = self.device
        self._sample = torch.zeros(batch, e.in_ch, height, width, dtype=torch.float32, device=dev)
        self._t = torch.zeros(batch, dtype=torch.float32, device=dev)
        self._ctx = torch.zeros(batch, d_ctx, 1, seq_len, dtype=torch.float16, device=dev)
        self._time_ids = (torch.zeros(spec["time_ids"]["shape"], dtype=torch.float32, device=dev) if e.xl else None)
        self._text_embeds = (torch.zeros(spec["text_embeds"]["shape"], dtype=torch.float32, device=dev)
                             if e.xl else None)
        self._res = [torch.zeros(s, dtype=torch.float16, device=dev) for s in self.res_shapes]
        self._cond = (torch.zeros(batch, e.time_cond_dim, dtype=torch.float32, device=dev) if e.time_cond_dim
                      else None)
        self._out = torch.zeros(batch, e.out_ch, height, width, dtype=torch.float32, device=dev)
        # device-resident loop (pipeline.denoise): the UNet input as the kernels read it (NHWC fp16, written by the
        # fused CFG + scheduler kernel), the per-prompt cross-attention K/V, the conv_out epilogue's NHWC output
        self._x_nhwc = torch.zeros(batch, height, width, e.in_pad, dtype=torch.float16, device=dev)
        self._kv_all = (torch.zeros(batch * seq_len, e.kv_total, dtype=torch.float16, device=dev)
                        if e.kv_w is not None else None)
        self._out_nhwc = torch.zeros(batch, height, width, e.out_ch, dtype=torch.float32, device=dev)
        self._graph = None
        self.use_cuda_graph = use_cuda_graph
        self.launches_per_call = None

    def residual_shapes(self):
        """NCHW shapes of the 13 ControlNet residuals (controlnet.py:218-229 order)."""
        e = self.engine
        shapes = [(self.batch, e.boc[0], self.h, self.w)]
        h, w = self.h, self.w
        for i, c in enumerate(e.boc):
            for _ in range(e.lpb):
                shapes.append((self.batch, c, h, w))
            if i != e.nb - 1:
                h, w = h // 2, w // 2
                shapes.append((self.batch, c, h, w))
        shapes.append((self.batch, e.boc[-1], h, w))
        return shapes

    # -- device-side sequence (captured) --------------------------------------------------------
    def _run(self, rows=None):
        e = self.engine
        r = rows or self.batch
        x = L.nchw_to_nhwc(self._sample[:r], c_pad=e.in_pad)
        ctx = L.ctx_to_tokens(self._ctx[:r])
        res = [L.nchw_to_nhwc(b[:r]) for b in self._res] if self._res else None
        tid = self._time_ids[:r] if e.xl else None
        te = self._text_embeds[:r] if e.xl else None
        cond = self._cond[:r] if self._cond is not None else None
        out = e.forward(x, self._t[:r], ctx, self.seq, tid, te, res, timestep_cond=cond)
        L.nhwc_to_nchw_f32(out, c=e.out_ch, out=self._out[:r])

    # -- per-prompt prologue + per-step core of the device loop (pipeline.denoise) ------------------------------
    def prepare_prompt(self, rows=None):
        """Cross-attention keys / values of every block from ``_ctx`` (constant over the denoising loop)."""
        if self._kv_all is not None:
            r = rows or self.batch
            self.engine.kv_project(L.ctx_to_tokens(self._ctx[:r]), out=self._kv_all[:r * self.seq])

    def time_table(self, ts_rows, rows=None):
        """ts_rows: fp32 device tensor [n_steps * rows] (each step's timestep repeated per batch row) ->
        [n_steps, rows, sum Cout] time-embedding biases of every ResNet block for ALL steps (unet.py:442,476-478
        depend on t only): one small-M pass per 32 rows instead of three launches inside every step.  A
        guidance-embedding UNet reads the first ``rows`` rows of ``_cond``."""
        e, b = self.engine, rows or self.batch
        n_steps = ts_rows.shape[0] // b
        per = max(1, 32 // b)
        parts = []
        for s0 in range(0, n_steps, per):
            k = min(per, n_steps - s0)
            tid = self._time_ids[:b].repeat(k, 1) if e.xl else None
            te = self._text_embeds[:b].repeat(k, 1) if e.xl else None
            cond = self._cond[:b].repeat(k, 1) if self._cond is not None else None
            parts.append(e.time_embedding(ts_rows[s0 * b:(s0 + k) * b].contiguous(), tid, te, cond))
        return torch.cat(parts, 0).reshape(n_steps, b, -1)

    def _run_core(self, temb, residuals=None, rows=None):
        """One UNet forward on ``_x_nhwc`` with precomputed time-embedding biases ``temb`` [rows, sum Cout] and the
        prologue's K/V; the conv_out epilogue writes ``_out_nhwc``."""
        if rows is None or rows == self.batch:
            self.engine.forward(self._x_nhwc, None, None, self.seq, additional_residuals=residuals, temb_all=temb,
                                kv_all=self._kv_all, out=self._out_nhwc)
            return
        kv = self._kv_all[:rows * self.seq] if self._kv_all is not None else None
        self.engine.forward(self._x_nhwc[:rows], None, None, self.seq, additional_residuals=residuals,
                            temb_all=temb, kv_all=kv, out=self._out_nhwc[:rows])

    def _launch(self, rows=None):
        if rows is not None and rows != self.batch:  # the step-by-step guidance-free loop: eager, no graph of its own
            self._run(rows)
            return
        if not self.use_cuda_graph:
            self._run()
            return
        if self._graph is None:
            # warm-up on a side stream (one-time attribute / workspace setup must not be captured)
            s = torch.cuda.Stream(device=self.device)
            s.wait_stream(torch.cuda.current_stream())
            with torch.cuda.stream(s):
                n0 = L.launch_count()
                self._run()
                self.launches_per_call = L.launch_count() - n0
            torch.cuda.current_stream().wait_stream(s)
            torch.cuda.synchronize()
            g = torch.cuda.CUDAGraph()
            with torch.cuda.graph(g):
                self._run()
            self._graph = g
        self._graph.replay()

    def forward_device(self, sample, timestep, encoder_hidden_states, time_ids=None, text_embeds=None,
                       additional_residuals=None, timestep_cond=None):
        """CUDA tensors in, CUDA fp32 ``noise_pred`` (a view of the static output buffer) out.  ``sample`` may have
        fewer rows than the batch the model was built for (the guidance-free loop): then every input has that many
        rows and only those run."""
        r = sample.shape[0]
        if not 0 < r <= self.batch:
            raise ValueError(f"sample has {r} rows, the UNet was built for at most {self.batch}")
        self._sample[:r].copy_(sample)
        self._t[:r].copy_(timestep)
        self._ctx[:r].copy_(encoder_hidden_states)
        if self.engine.xl:
            self._time_ids[:r].copy_(time_ids.reshape(r, -1))
            self._text_embeds[:r].copy_(text_embeds)
        if self._cond is not None:
            if timestep_cond is None:
                raise ValueError(f"this UNet has time_cond_proj_dim={self.engine.time_cond_dim}: pass timestep_cond")
            self._cond[:r].copy_(timestep_cond)
        for buf, res in zip(self._res, additional_residuals or []):
            buf[:r].copy_(res)
        self._launch(r)
        return self._out[:r]

    def __call__(self, **kwargs):
        self._verify_inputs(**kwargs)
        missing = [k for k in self.expected_inputs if k not in kwargs]
        if missing:
            raise ValueError(f"Missing inputs: {missing}")
        as_numpy = isinstance(kwargs["sample"], np.ndarray)
        self._to_device(kwargs["sample"], self._sample)
        self._to_device(kwargs["timestep"], self._t)
        self._to_device(kwargs["encoder_hidden_states"], self._ctx)
        if self.engine.xl:
            self._to_device(kwargs["time_ids"], self._time_ids)
            self._to_device(kwargs["text_embeds"], self._text_embeds)
        if self._cond is not None:
            self._to_device(kwargs["timestep_cond"], self._cond)
        for i, buf in enumerate(self._res):
            self._to_device(kwargs[f"additional_residual_{i}"], buf)
        self._launch()
        if as_numpy:
            return {"noise_pred": self._out.cpu().numpy()}
        return {"noise_pred": self._out.clone()}
