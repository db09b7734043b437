"""UNet denoiser on the sm_90a kernels: weight pre-packing + the launch graph.

This is the device-side replacement for the traced graph of the reference
``UNet2DConditionModel.forward`` / ``UNet2DConditionModelXL.forward``
(``python_coreml_stable_diffusion/unet.py:975-1048``, ``:1051-1152``) that Core ML executes behind
``CoreMLModel.__call__``.  Layout is channels-last fp16 end to end: an NHWC image *is* the
token-major ``[B*H*W, C]`` matrix, so the reference's ``view(B, C, 1, H*W)`` (``unet.py:558``) is
free.  Every op is a call into ``libb200sd.so`` (``include/b200sd.h``); nothing here computes
with torch.

Pre-packing (done once at load):
  * 3x3 conv ``[Co, Ci, 3, 3]`` -> ``[Co, 9*Ci]`` (OHWI); ``conv_in`` input channels padded 4 -> 8;
  * 1x1 conv / linear -> ``[Co, Ci]``; self-attention ``to_q|to_k|to_v`` fused to ``[3C, C]``;
  * every cross-attention ``to_k|to_v`` of the whole net concatenated to one ``[sum 2C, D_ctx]``
    matrix (the text states are the same for all 16 blocks: one GEMM instead of 32);
  * GEGLU projection rows interleaved (value_i, gate_i) so the gate product is a GEMM epilogue;
  * all ``time_emb_proj`` matrices concatenated (+ ``conv1`` bias folded in): one small-M kernel
    yields the per-image bias vectors of all ResNet blocks.
"""
from __future__ import annotations

import enum
import os

import torch

from . import lib as L


class AttentionImplementations(enum.Enum):
    """Mirror of the reference switch (``unet.py:33-39``).  All three names select the same fused
    flash kernel (they are one mathematical function, ``attention.py:24-168``); the value is passed
    down as the kernel's tile-policy hint."""
    ORIGINAL = "ORIGINAL"
    SPLIT_EINSUM = "SPLIT_EINSUM"
    SPLIT_EINSUM_V2 = "SPLIT_EINSUM_V2"


ATTENTION_IMPLEMENTATION_IN_EFFECT = AttentionImplementations.SPLIT_EINSUM
_IMPL_CODE = {AttentionImplementations.ORIGINAL: 0, AttentionImplementations.SPLIT_EINSUM: 1,
              AttentionImplementations.SPLIT_EINSUM_V2: 2}


def _as_list(v, n):
    return list(v) if isinstance(v, (list, tuple)) else [v] * n


def _w2d(sd, key):
    w = sd[key]
    return w.reshape(w.shape[0], -1) if w.dim() == 4 and w.shape[2] == 1 else w


class _Packer:
    def __init__(self, sd, device):
        self.sd = sd
        self.dev = device

    def f16(self, t):
        return t.detach().to(device=self.dev, dtype=torch.float16).contiguous()

    def f32(self, key):
        return self.sd[key].detach().to(device=self.dev, dtype=torch.float32).contiguous()

    def conv3(self, key, pad_in=None):
        w = self.sd[key + ".weight"].detach().float()
        if pad_in is not None and w.shape[1] < pad_in:
            w = torch.nn.functional.pad(w, (0, 0, 0, 0, 0, pad_in - w.shape[1]))
        return self.f16(w.permute(0, 2, 3, 1).reshape(w.shape[0], -1))

    def lin(self, key):
        return self.f16(_w2d(self.sd, key + ".weight").float())

    def bias(self, key):
        k = key + ".bias"
        return self.f32(k) if k in self.sd else None


class UNetEngine:
    """Holds device-resident packed weights and issues the forward launch sequence."""

    def __init__(self, cfg: dict, state_dict: dict, device="cuda"):
        L.load()
        self.cfg = dict(cfg)
        self.dev = torch.device(device)
        boc = list(cfg["block_out_channels"])
        nb = len(boc)
        self.boc, self.nb = boc, nb
        self.lpb = cfg.get("layers_per_block", 2)
        self.heads = _as_list(cfg.get("attention_head_dim", 8), nb)
        self.depth = _as_list(cfg.get("transformer_layers_per_block", 1), nb)
        self.mid_depth = cfg.get("mid_block_transformer_layers", self.depth[-1])
        self.groups = cfg.get("norm_num_groups", 32)
        self.eps = cfg.get("norm_eps", 1e-5)
        self.down_types = list(cfg["down_block_types"])
        self.up_types = list(cfg["up_block_types"])
        self.in_ch = cfg.get("in_channels", 4)
        self.out_ch = cfg.get("out_channels", 4)
        self.in_pad = max(8, (self.in_ch + 7) // 8 * 8)
        self.xl = cfg.get("addition_embed_type") == "text_time"
        self.support_controlnet = bool(cfg.get("support_controlnet", False))
        # Normalisation fusion level (B200SD_FUSED):
        #   "ln" (default)  LayerNorm folded into its consumer GEMM, row statistics from the producer's epilogue;
        #                   GroupNorm stays the one-launch cluster kernel in front of the 9-tap TMA convolution (the
        #                   fused-GroupNorm variants below are opt-in; they have not been timed against it on H100)
        #   "1"  GroupNorm + SiLU applied in the halo convolution's operand path (no GroupNorm launch at all),
        #        statistics from the producers' staged epilogues
        #   "2"  statistics from the producers, one elementwise GroupNorm-apply launch + 9-tap convolution
        #   "3"  "1" on maps of >= B200SD_HALO_MIN_HW pixels, "2" below
        #   "0"  round-1 graph (standalone GroupNorm and LayerNorm launches)
        fm = os.environ.get("B200SD_FUSED", "ln")
        self.fused = fm != "0"
        self.fuse_gn = fm in ("1", "2", "3")
        self.halo_min_hw = {"1": 0, "2": 1 << 30, "3": int(os.environ.get("B200SD_HALO_MIN_HW", "1024"))}.get(fm, 1 << 30)
        # plain stride-1 3x3 convolutions on maps of at least this many pixels take the halo-reuse kernel with TMA patches
        # (lib.conv3x3(halo=2)); smaller maps keep the 9-tap form, whose split-K fills the GPU.  0 disables.
        self.halo_tma_min_hw = int(os.environ.get("B200SD_HALO_TMA", "0"))
        # ResNet shortcuts (1x1 convolutions on the block input) run as extra k-blocks of conv2 instead of their own launch
        self.fold_shortcut = os.environ.get("B200SD_FOLD_SC", "1") != "0"
        for c, h in zip(boc, self.heads):
            if c % h or c // h != 64:
                raise L.B200SDError(f"b200sd attention kernel needs head dim 64 (got {c}/{h})")
        self._pack(state_dict)

    # ------------------------------------------------------------------ packing
    def _pack(self, sd):
        P = _Packer(sd, self.dev)
        w = {}
        self.temb_slices = {}   # resnet prefix -> (offset, cout)
        temb_w, temb_b = [], []
        self.kv_slices = {}     # attn2 prefix -> (offset, C)
        kv_w = []
        off_t = off_kv = 0

        def resnet(p):
            nonlocal off_t
            r = {"n1g": P.f32(p + ".norm1.weight"), "n1b": P.f32(p + ".norm1.bias"),
                 "c1": P.conv3(p + ".conv1"),
                 "n2g": P.f32(p + ".norm2.weight"), "n2b": P.f32(p + ".norm2.bias"),
                 "c2": P.conv3(p + ".conv2"), "c2b": P.bias(p + ".conv2")}
            co = r["c1"].shape[0]
            temb_w.append(_w2d(sd, p + ".time_emb_proj.weight").float())
            temb_b.append(sd[p + ".time_emb_proj.bias"].float() + sd[p + ".conv1.bias"].float())
            self.temb_slices[p] = (off_t, co)
            off_t += co
            if (p + ".conv_shortcut.weight") in sd:
                r["sc"] = P.lin(p + ".conv_shortcut")
                r["scb"] = P.bias(p + ".conv_shortcut")
                # the shortcut folded into conv2: its [Cout, Cin] matrix appended along K (extra centre-tap k-blocks of
                # the same convolution launch, lib.conv3x3(shortcut=...)), one bias vector for both
                if self.fold_shortcut and not self.fuse_gn and self.fused:
                    r["c2sc"] = torch.cat([r["c2"], r["sc"]], 1).contiguous()
                    r["c2scb"] = (r["c2b"] + r["scb"]).contiguous()
            w[p] = r

        def transformer(p, c, depth):
            nonlocal off_kv
            t = {"ng": P.f32(p + ".norm.weight"), "nb": P.f32(p + ".norm.bias"),
                 "pi": P.lin(p + ".proj_in"), "pib": P.bias(p + ".proj_in"),
                 "po": P.lin(p + ".proj_out"), "pob": P.bias(p + ".proj_out"), "blocks": []}
            for d in range(depth):
                b = f"{p}.transformer_blocks.{d}"
                blk = {}
                for i in (1, 2, 3):
                    blk[f"ln{i}g"] = P.f32(f"{b}.norm{i}.weight")
                    blk[f"ln{i}b"] = P.f32(f"{b}.norm{i}.bias")
                blk["qkv"] = P.f16(torch.cat([_w2d(sd, f"{b}.attn1.to_{n}.weight").float() for n in "qkv"], 0))
                blk["o1"], blk["o1b"] = P.lin(f"{b}.attn1.to_out.0"), P.bias(f"{b}.attn1.to_out.0")
                blk["q2"] = P.lin(f"{b}.attn2.to_q")
                kv_w.append(torch.cat([_w2d(sd, f"{b}.attn2.to_k.weight").float(),
                                       _w2d(sd, f"{b}.attn2.to_v.weight").float()], 0))
                blk["kv_off"] = off_kv
                off_kv += 2 * c
                blk["o2"], blk["o2b"] = P.lin(f"{b}.attn2.to_out.0"), P.bias(f"{b}.attn2.to_out.0")
                gw = _w2d(sd, f"{b}.ff.net.0.proj.weight").float()
                gb = sd[f"{b}.ff.net.0.proj.bias"].float()
                half = gw.shape[0] // 2
                blk["gg"] = P.f16(torch.stack([gw[:half], gw[half:]], 1).reshape(gw.shape))
                blk["ggb"] = torch.stack([gb[:half], gb[half:]], 1).reshape(-1).to(self.dev).contiguous()
                blk["f2"], blk["f2b"] = P.lin(f"{b}.ff.net.2"), P.bias(f"{b}.ff.net.2")
                if self.fused:
                    # LayerNorm folded into the consumer GEMM (layer_norm.py:66-78 followed by unet.py:74-82 / :613):
                    # W' = gamma (.) W (fp16), wg = row sums of the ROUNDED W', bias' = W beta + bias
                    for name, ln, bkey in (("qkv", 1, None), ("q2", 2, None), ("gg", 3, "ggb")):
                        wf32 = blk[name].float()
                        folded = (wf32 * blk[f"ln{ln}g"][None, :]).half().contiguous()
                        blk[name + "_ln"] = folded
                        blk[name + "_wg"] = folded.float().sum(1).contiguous()
                        bias = wf32 @ blk[f"ln{ln}b"]
                        if bkey is not None:
                            bias = bias + blk[bkey]
                        blk[name + "_lnb"] = bias.contiguous()
                t["blocks"].append(blk)
            w[p] = t

        boc, nb, lpb = self.boc, self.nb, self.lpb
        w["conv_in"] = {"w": P.conv3("conv_in", pad_in=self.in_pad), "b": P.bias("conv_in")}
        w["time"] = {"l1": P.lin("time_embedding.linear_1"), "l1b": P.bias("time_embedding.linear_1"),
                     "l2": P.lin("time_embedding.linear_2"), "l2b": P.bias("time_embedding.linear_2")}
        if self.xl:
            w["add"] = {"l1": P.lin("add_embedding.linear_1"), "l1b": P.bias("add_embedding.linear_1"),
                        "l2": P.lin("add_embedding.linear_2"), "l2b": P.bias("add_embedding.linear_2")}
        for i, typ in enumerate(self.down_types):
            for j in range(lpb):
                resnet(f"down_blocks.{i}.resnets.{j}")
                if typ == "CrossAttnDownBlock2D":
                    transformer(f"down_blocks.{i}.attentions.{j}", boc[i], self.depth[i])
            if i != nb - 1:
                p = f"down_blocks.{i}.downsamplers.0.conv"
                w[p] = {"w": P.conv3(p), "b": P.bias(p)}
        resnet("mid_block.resnets.0")
        transformer("mid_block.attentions.0", boc[-1], self.mid_depth)
        resnet("mid_block.resnets.1")
        rboc, rdepth = boc[::-1], self.depth[::-1]
        for i, typ in enumerate(self.up_types):
            for j in range(lpb + 1):
                resnet(f"up_blocks.{i}.resnets.{j}")
                if typ == "CrossAttnUpBlock2D":
                    transformer(f"up_blocks.{i}.attentions.{j}", rboc[i], rdepth[i])
            if i != nb - 1:
                p = f"up_blocks.{i}.upsamplers.0.conv"
                w[p] = {"w": P.conv3(p), "b": P.bias(p)}
        w["out"] = {"g": P.f32("conv_norm_out.weight"), "b": P.f32("conv_norm_out.bias"),
                    "w": P.conv3("conv_out"), "cb": P.bias("conv_out")}
        self.temb_w = P.f16(torch.cat(temb_w, 0))
        self.temb_b = torch.cat(temb_b, 0).to(self.dev).contiguous()
        self.temb_total = off_t
        self.kv_w = P.f16(torch.cat(kv_w, 0)) if kv_w else None
        self.kv_total = off_kv
        self.w = w
        self.weight_bytes = sum(t.numel() * t.element_size() for t in self._tensors())

    def _tensors(self):
        def walk(o):
            if torch.is_tensor(o):
                yield o
            elif isinstance(o, dict):
                for v in o.values():
                    yield from walk(v)
            elif isinstance(o, list):
                for v in o:
                    yield from walk(v)
        yield from walk(self.w)
        yield self.temb_w
        yield self.temb_b
        if self.kv_w is not None:
            yield self.kv_w

    # ------------------------------------------------------------------ blocks
    def _resnet(self, p, x, x1, temb_all):
        r = self.w[p]
        n, h, wd, _ = x.shape
        off, co = self.temb_slices[p]
        hh = L.group_norm(x, r["n1g"], r["n1b"], self.groups, self.eps, silu=True, x1=x1)
        hh = L.conv3x3(hh, r["c1"], temb_all[:, off:], bias_rows=h * wd, bias_stride=self.temb_total)
        hh = L.group_norm(hh, r["n2g"], r["n2b"], self.groups, self.eps, silu=True)
        if "sc" in r:
            res = L.linear(x.reshape(n * h * wd, -1), r["sc"], r["scb"],
                           x1=None if x1 is None else x1.reshape(n * h * wd, -1), static_w=True)
        else:
            res = x
        return L.conv3x3(hh, r["c2"], r["c2b"], res)

    def _transformer(self, p, x, kv_all, batch, heads, s_ctx):
        t = self.w[p]
        n, h, wd, c = x.shape
        m, s = n * h * wd, h * wd
        impl = _IMPL_CODE[ATTENTION_IMPLEMENTATION_IN_EFFECT]
        hn = L.group_norm(x, t["ng"], t["nb"], 32, 1e-6, silu=False)
        tok = L.linear(hn.reshape(m, c), t["pi"], t["pib"], static_w=True)
        for blk in t["blocks"]:
            n1 = L.layer_norm(tok, blk["ln1g"], blk["ln1b"])
            qkv = L.linear(n1, blk["qkv"], static_w=True)
            a = L.attention(qkv[:, :c], qkv[:, c:2 * c], qkv[:, 2 * c:], batch, heads, s, s, impl=impl)
            tok = L.linear(a, blk["o1"], blk["o1b"], tok, static_w=True)
            n2 = L.layer_norm(tok, blk["ln2g"], blk["ln2b"])
            q = L.linear(n2, blk["q2"], static_w=True)
            ko = blk["kv_off"]
            a = L.attention(q, kv_all[:, ko:ko + c], kv_all[:, ko + c:ko + 2 * c], batch, heads, s, s_ctx, impl=impl)
            tok = L.linear(a, blk["o2"], blk["o2b"], tok, static_w=True)
            n3 = L.layer_norm(tok, blk["ln3g"], blk["ln3b"])
            g = L.linear(n3, blk["gg"], blk["ggb"], geglu=True, static_w=True)
            tok = L.linear(g, blk["f2"], blk["f2b"], tok, static_w=True)
        out = L.linear(tok, t["po"], t["pob"], x.reshape(m, c), static_w=True)
        return out.reshape(n, h, wd, c)

    # ------------------------------------------------------------------ fused blocks
    # An activation travels as (tensor, chan): chan = per-channel (sum, sum of squares) [n, C, 2] left behind by the
    # epilogue that produced the tensor, or None when the producer could not emit them (then the consumer falls back
    # to the standalone GroupNorm kernel).
    def _use_halo(self, x):
        return x.shape[1] * x.shape[2] >= self.halo_min_hw

    def _halo_tma(self, x, wgt, kw=None):
        """2 (halo reuse with TMA patches) for a plain fp16 stride-1 convolution on a large enough map, else False."""
        kw = kw or {}
        ok = (self.halo_tma_min_hw > 0 and x.shape[1] * x.shape[2] >= self.halo_tma_min_hw and wgt.shape[0] % 32 == 0
              and kw.get("stride", 1) == 1 and kw.get("out_dtype", torch.float16) == torch.float16 and not kw.get("act"))
        return 2 if ok else False

    def _gn_conv(self, x, xs, x1, x1s, gamma, beta, eps, silu, wgt, bias, residual=None, stats=None, **kw):
        if not self.fuse_gn:  # standalone GroupNorm launch + plain convolution, no statistics side outputs
            hh = L.group_norm(x, gamma, beta, self.groups, eps, silu=silu, x1=x1)
            return L.conv3x3(hh, wgt, bias, residual, halo=False if kw.get("shortcut") else self._halo_tma(hh, wgt, kw), **kw)
        have = xs is not None and (x1 is None or x1s is not None)
        halo = self._use_halo(x)
        if have and halo:
            gn = dict(chan0=xs, chan1=x1s, gamma=gamma, beta=beta, groups=self.groups, eps=eps, silu=silu)
            return L.conv3x3(x, wgt, bias, residual, x1=x1, halo=True, gn=gn, stats=stats, **kw)
        if have:
            hh = L.group_norm_apply(x, xs, gamma, beta, self.groups, eps, silu=silu, x1=x1, chan1=x1s)
        else:
            hh = L.group_norm(x, gamma, beta, self.groups, eps, silu=silu, x1=x1)
        return L.conv3x3(hh, wgt, bias, residual, halo=halo, stats=stats, **kw)

    def _resnet_f(self, p, x, xs, x1, x1s, temb_all):
        r = self.w[p]
        n, h, wd, _ = x.shape
        off, co = self.temb_slices[p]
        st1, st2 = {}, {}
        hh = self._gn_conv(x, xs, x1, x1s, r["n1g"], r["n1b"], self.eps, True, r["c1"], temb_all[:, off:],
                           stats=st1 if self.fuse_gn else None, bias_rows=h * wd, bias_stride=self.temb_total)
        if "c2sc" in r:
            # out = conv2(h) + conv_shortcut(x ++ x1) as ONE launch (unet.py:483-489)
            out = self._gn_conv(hh, None, None, None, r["n2g"], r["n2b"], self.eps, True, r["c2sc"], r["c2scb"], None,
                                shortcut=(x, x1))
            return out, None
        if "sc" in r:
            res = L.linear(x.reshape(n * h * wd, -1), r["sc"], r["scb"],
                           x1=None if x1 is None else x1.reshape(n * h * wd, -1), static_w=True)
        else:
            res = x
        out = self._gn_conv(hh, st1.get("chan"), None, None, r["n2g"], r["n2b"], self.eps, True, r["c2"], r["c2b"], res,
                            stats=st2 if self.fuse_gn else None)
        return out, st2.get("chan")

    def _transformer_f(self, p, x, xs, kv_all, batch, heads, s_ctx):
        t = self.w[p]
        n, h, wd, c = x.shape
        m, s = n * h * wd, h * wd
        impl = _IMPL_CODE[ATTENTION_IMPLEMENTATION_IN_EFFECT]
        rs = {}
        if self.fuse_gn and xs is not None and self._use_halo(x):
            gn = dict(chan0=xs, chan1=None, gamma=t["ng"], beta=t["nb"], groups=32, eps=1e-6, silu=False)
            tok = L.conv3x3(x, t["pi"], t["pib"], halo=True, taps=1, gn=gn, rowstats=rs).reshape(m, c)
        else:
            hn = (L.group_norm_apply(x, xs, t["ng"], t["nb"], 32, 1e-6) if (self.fuse_gn and xs is not None)
                  else L.group_norm(x, t["ng"], t["nb"], 32, 1e-6, silu=False))
            tok = L.linear(hn.reshape(m, c), t["pi"], t["pib"], static_w=True, rowstats=rs)

        def ln_of(rs, blk, name):
            return dict(stat=rs["rows"], parts=rs["parts"], wg=blk[name + "_wg"], eps=1e-5)

        nblk = len(t["blocks"])
        for bi, blk in enumerate(t["blocks"]):
            qkv = L.linear(tok, blk["qkv_ln"], blk["qkv_lnb"], ln=ln_of(rs, blk, "qkv"), static_w=True)
            a = L.attention(qkv[:, :c], qkv[:, c:2 * c], qkv[:, 2 * c:], batch, heads, s, s, impl=impl)
            rs = {}
            tok = L.linear(a, blk["o1"], blk["o1b"], tok, static_w=True, rowstats=rs)
            q = L.linear(tok, blk["q2_ln"], blk["q2_lnb"], ln=ln_of(rs, blk, "q2"), static_w=True)
            ko = blk["kv_off"]
            a = L.attention(q, kv_all[:, ko:ko + c], kv_all[:, ko + c:ko + 2 * c], batch, heads, s, s_ctx, impl=impl)
            rs = {}
            tok = L.linear(a, blk["o2"], blk["o2b"], tok, static_w=True, rowstats=rs)
            g = L.linear(tok, blk["gg_ln"], blk["gg_lnb"], geglu=True, ln=ln_of(rs, blk, "gg"), static_w=True)
            rs = {}
            tok = L.linear(g, blk["f2"], blk["f2b"], tok, static_w=True, rowstats=rs if bi + 1 < nblk else None)
        st = {}
        ok = self.fuse_gn and (s % 128 == 0 or (s >= 16 and 128 % s == 0))   # geometries whose tiles map onto whole images
        out = L.linear(tok, t["po"], t["pob"], x.reshape(m, c), static_w=True, stats=st if ok else None, cs_hw=s)
        return out.reshape(n, h, wd, c), st.get("chan")

    def _forward_fused(self, sample, temb_all, kv_all, batch, s_ctx, additional_residuals, out=None):
        st = {}
        x = L.conv3x3(sample, self.w["conv_in"]["w"], self.w["conv_in"]["b"], stats=st if self.fuse_gn else None)
        xs = st.get("chan")
        skips = [(x, xs)]
        for i, typ in enumerate(self.down_types):
            for j in range(self.lpb):
                x, xs = self._resnet_f(f"down_blocks.{i}.resnets.{j}", x, xs, None, None, temb_all)
                if typ == "CrossAttnDownBlock2D":
                    x, xs = self._transformer_f(f"down_blocks.{i}.attentions.{j}", x, xs, kv_all, batch, self.heads[i], s_ctx)
                skips.append((x, xs))
            if i != self.nb - 1:
                d = self.w[f"down_blocks.{i}.downsamplers.0.conv"]
                st = {}
                x = L.conv3x3(x, d["w"], d["b"], stride=2, stats=st if self.fuse_gn else None)
                xs = st.get("chan")
                skips.append((x, xs))
        if additional_residuals is not None:  # the sums have no producer-side statistics: standalone GroupNorm there
            skips = [(L.add(s, r), None) for (s, _), r in zip(skips, additional_residuals[:-1])]
        x, xs = self._resnet_f("mid_block.resnets.0", x, xs, None, None, temb_all)
        x, xs = self._transformer_f("mid_block.attentions.0", x, xs, kv_all, batch, self.heads[-1], s_ctx)
        x, xs = self._resnet_f("mid_block.resnets.1", x, xs, None, None, temb_all)
        if additional_residuals is not None:
            x, xs = L.add(x, additional_residuals[-1]), None
        rheads = self.heads[::-1]
        for i, typ in enumerate(self.up_types):
            for j in range(self.lpb + 1):
                sk, sks = skips.pop()
                x, xs = self._resnet_f(f"up_blocks.{i}.resnets.{j}", x, xs, sk, sks, temb_all)
                if typ == "CrossAttnUpBlock2D":
                    x, xs = self._transformer_f(f"up_blocks.{i}.attentions.{j}", x, xs, kv_all, batch, rheads[i], s_ctx)
            if i != self.nb - 1:
                u = self.w[f"up_blocks.{i}.upsamplers.0.conv"]
                st = {}
                if self.fuse_gn and 4 * x.shape[1] * x.shape[2] >= self.halo_min_hw:
                    x = L.conv3x3(x, u["w"], u["b"], halo=True, upsample=True, stats=st)
                else:
                    up = L.upsample2x(x)
                    x = L.conv3x3(up, u["w"], u["b"], stats=st if self.fuse_gn else None,
                                  halo=False if self.fuse_gn else self._halo_tma(up, u["w"]))
                xs = st.get("chan")
        o = self.w["out"]
        return self._gn_conv(x, xs, None, None, o["g"], o["b"], self.eps, True, o["w"], o["cb"], out_dtype=torch.float32,
                             out=out)

    # ------------------------------------------------------------------ forward
    def time_embedding(self, timesteps, time_ids=None, text_embeds=None):
        """fp32 [B] -> per-image bias vectors of every ResNet block: fp32 [B, sum Cout]."""
        cfg = self.cfg
        tw = self.w["time"]
        t_emb = L.timestep_embedding(timesteps, self.boc[0], cfg.get("flip_sin_to_cos", True),
                                     cfg.get("freq_shift", 0))
        emb = L.linear_small(L.linear_small(t_emb, tw["l1"], tw["l1b"], act_out=True), tw["l2"], tw["l2b"])
        if self.xl:
            aw = self.w["add"]
            te = L.timestep_embedding(time_ids.reshape(-1).float().contiguous(), cfg["addition_time_embed_dim"],
                                      cfg.get("flip_sin_to_cos", True), cfg.get("freq_shift", 0))
            add_in = torch.cat([text_embeds.float(), te.reshape(text_embeds.shape[0], -1)], dim=-1).contiguous()
            aug = L.linear_small(L.linear_small(add_in, aw["l1"], aw["l1b"], act_out=True), aw["l2"], aw["l2b"])
            emb = emb + aug
        return L.linear_small(emb, self.temb_w, self.temb_b, act_in=True)

    def kv_project(self, ctx_tokens, out=None):
        """to_k | to_v of every cross-attention block on the text states (unet.py:79-82): one GEMM.  The text states
        do not change during a denoising loop, so the pipeline calls this once per prompt, not once per step."""
        return L.linear(ctx_tokens, self.kv_w, static_w=True, out=out) if self.kv_w is not None else None

    def forward(self, sample, timesteps, ctx_tokens, s_ctx, time_ids=None, text_embeds=None,
                additional_residuals=None, temb_all=None, kv_all=None, out=None):
        """sample: NHWC fp16 [B, H, W, in_pad]; timesteps fp32 [B]; ctx_tokens fp16 [B*s_ctx, D].
        additional_residuals: list of NHWC fp16 tensors (ControlNet, unet.py:1009-1022).
        temb_all / kv_all: precomputed time-embedding biases [B, sum Cout] / cross-attention keys and values (the
        per-prompt prologue of the pipeline's loop); out: optional fp32 NHWC output buffer.
        Returns noise_pred NHWC fp32 [B, H, W, out_ch]."""
        batch = sample.shape[0]
        if temb_all is None:
            temb_all = self.time_embedding(timesteps, time_ids, text_embeds)
        if kv_all is None:
            kv_all = self.kv_project(ctx_tokens)
        if self.fused:
            return self._forward_fused(sample, temb_all, kv_all, batch, s_ctx, additional_residuals, out)
        x = L.conv3x3(sample, self.w["conv_in"]["w"], self.w["conv_in"]["b"])
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
        if additional_residuals is not None:
            skips = [L.add(s, r) for s, r in zip(skips, additional_residuals[:-1])]
        x = self._resnet("mid_block.resnets.0", x, None, temb_all)
        x = self._transformer("mid_block.attentions.0", x, kv_all, batch, self.heads[-1], s_ctx)
        x = self._resnet("mid_block.resnets.1", x, None, temb_all)
        if additional_residuals is not None:
            x = L.add(x, additional_residuals[-1])
        rheads = self.heads[::-1]
        for i, typ in enumerate(self.up_types):
            for j in range(self.lpb + 1):
                x = self._resnet(f"up_blocks.{i}.resnets.{j}", x, skips.pop(), temb_all)
                if typ == "CrossAttnUpBlock2D":
                    x = self._transformer(f"up_blocks.{i}.attentions.{j}", x, kv_all, batch, rheads[i], s_ctx)
            if i != self.nb - 1:
                u = self.w[f"up_blocks.{i}.upsamplers.0.conv"]
                x = L.conv3x3(L.upsample2x(x), u["w"], u["b"])
        o = self.w["out"]
        x = L.group_norm(x, o["g"], o["b"], self.groups, self.eps, silu=True)
        return L.conv3x3(x, o["w"], o["cb"], out_dtype=torch.float32, out=out)
