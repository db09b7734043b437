"""Plain-PyTorch fp32 restatement of the reference hot path.  TEST INFRASTRUCTURE ONLY.

Functional (state-dict driven) NCHW restatement of:

* ``UNet2DConditionModel.forward`` / ``UNet2DConditionModelXL.forward``
  (reference ``python_coreml_stable_diffusion/unet.py:975-1048`` and ``:1051-1152``)
  including ``ResnetBlock2D`` (:470-489), ``SpatialTransformer`` (:553-563),
  ``BasicTransformerBlock`` (:586-591), ``CrossAttention`` (:87-118), ``GEGLU`` (:616-617),
  ``get_timestep_embedding`` (:703-728), ``TimestepEmbedding`` (:665-682),
  ``Upsample2D``/``Downsample2D`` (:492-510), ControlNet residual injection (:1009-1022);
* the three attention variants of ``attention.py`` (``original`` :147-168,
  ``split_einsum`` :24-72, ``split_einsum_v2`` :75-144) -- mathematically one function;
* ``LayerNormANE`` (``layer_norm.py:51-80``), applied here in the *diffusers* convention
  ``x_hat * w + b`` because the reference's load hook (``unet.py:132-138``) divides the
  checkpoint bias by the weight so that ``(x_hat + b/w) * w`` is the same function;
* the VAE decoder and DDIM/DPM-Solver++/PNDM steps, whose arithmetic lives in un-vendored
  ``diffusers==0.30.2`` (call sites ``torch2coreml.py:584-594``, ``pipeline.py:565-569``);
  specs in SURVEY.md Appendix B; in-tree twins ``swift/StableDiffusion/pipeline/Scheduler.swift``
  and ``DPMSolverMultistepScheduler.swift``.

PIN STATUS
  UNet / attention / LayerNorm: pinned -- checked against the unmodified reference modules
  (``oracle.ref_unet``) in ``tests/test_oracle.py`` and via ``tests/golden/*.npz`` which
  were produced by the reference itself (``tests/golden/make_golden.py``).
  VAE decoder and scheduler steps: **parity unpinned** -- no runnable reference
  implementation or golden vector exists for them (diffusers is not installed and the Swift
  twins cannot be compiled); they are checked only against closed-form identities.

State dicts use diffusers key names (the reference's too, ``unet.py:121-146``); 1x1 conv /
linear weights may be 2-D or 4-D.
"""
from __future__ import annotations

import math

import torch
import torch.nn.functional as F


# --------------------------------------------------------------------------------------
# helpers
# --------------------------------------------------------------------------------------
def _f(t):
    """fp32, or fp64 when given fp64 (a state dict and inputs in fp64 run the whole restatement in fp64)."""
    return t if t.dtype == torch.float64 else t.float()


def _w(sd, key):
    return _f(sd[key])


def _conv(sd, prefix, x, stride=1, padding=0):
    w = _w(sd, prefix + ".weight")
    if w.dim() == 2:
        w = w[:, :, None, None]
    b = sd.get(prefix + ".bias")
    return F.conv2d(x, w, None if b is None else _f(b), stride=stride, padding=padding)


def _gn(sd, prefix, x, groups, eps):
    return F.group_norm(x, groups, _w(sd, prefix + ".weight"), _w(sd, prefix + ".bias"), eps)


def layer_norm_channels(x, weight, bias, eps=1e-5):
    """LayerNorm over the channel axis of a (B, C, 1, S) tensor, torch convention."""
    mu = x.mean(dim=1, keepdim=True)
    xc = x - mu
    var = (xc * xc).mean(dim=1, keepdim=True)
    y = xc * torch.rsqrt(var + eps)
    return y * weight.view(1, -1, 1, 1) + bias.view(1, -1, 1, 1)


def attention(q, k, v, heads, dim_head, mask=None):
    """softmax(q^T k / sqrt(d) [+ mask]) v on (B, C, 1, S) tensors; all three reference
    variants compute exactly this."""
    b = q.shape[0]
    qh = q.reshape(b, heads, dim_head, -1)
    kh = k.reshape(b, heads, dim_head, -1)
    vh = v.reshape(b, heads, dim_head, -1)
    s = torch.einsum("bhdq,bhdk->bhqk", qh, kh) * (dim_head ** -0.5)
    if mask is not None:  # additive, shape (B, Sk, 1, 1) as in unet.py:99-114
        s = s + mask.reshape(b, 1, 1, -1)
    p = s.softmax(dim=-1)
    o = torch.einsum("bhqk,bhdk->bhdq", p, vh)
    return o.reshape(b, heads * dim_head, 1, -1)


def timestep_embedding(timesteps, dim, flip_sin_to_cos=True, freq_shift=0.0, max_period=10000):
    half = dim // 2
    freqs = torch.exp(-math.log(max_period) * torch.arange(half, dtype=torch.float32, device=timesteps.device)
                      / (half - freq_shift))
    ang = _f(timesteps)[:, None] * freqs[None, :]
    s, c = torch.sin(ang), torch.cos(ang)
    return torch.cat([c, s], dim=-1) if flip_sin_to_cos else torch.cat([s, c], dim=-1)


# --------------------------------------------------------------------------------------
# UNet
# --------------------------------------------------------------------------------------
def _time_mlp(sd, prefix, x):
    h = _conv(sd, prefix + ".linear_1", x[:, :, None, None])
    return _conv(sd, prefix + ".linear_2", F.silu(h))


def _resnet(sd, p, x, temb, groups, eps):
    h = _conv(sd, p + ".conv1", F.silu(_gn(sd, p + ".norm1", x, groups, eps)), padding=1)
    if temb is not None and (p + ".time_emb_proj.weight") in sd:
        h = h + _conv(sd, p + ".time_emb_proj", F.silu(temb))
    h = _conv(sd, p + ".conv2", F.silu(_gn(sd, p + ".norm2", h, groups, eps)), padding=1)
    if (p + ".conv_shortcut.weight") in sd:
        x = _conv(sd, p + ".conv_shortcut", x)
    return x + h


def _cross_attn(sd, p, x, ctx, heads):
    q = _conv(sd, p + ".to_q", x)
    src = x if ctx is None else ctx
    k = _conv(sd, p + ".to_k", src)
    v = _conv(sd, p + ".to_v", src)
    d = q.shape[1] // heads
    return _conv(sd, p + ".to_out.0", attention(q, k, v, heads, d))


def _tblock(sd, p, x, ctx, heads):
    ln = lambda n, t: layer_norm_channels(t, _w(sd, f"{p}.{n}.weight"), _w(sd, f"{p}.{n}.bias"))
    x = _cross_attn(sd, p + ".attn1", ln("norm1", x), None, heads) + x
    x = _cross_attn(sd, p + ".attn2", ln("norm2", x), ctx, heads) + x
    a, g = _conv(sd, p + ".ff.net.0.proj", ln("norm3", x)).chunk(2, dim=1)
    x = _conv(sd, p + ".ff.net.2", a * F.gelu(g)) + x
    return x


def _spatial_transformer(sd, p, x, ctx, heads, depth):
    b, c, h, w = x.shape
    res = x
    t = _conv(sd, p + ".proj_in", _gn(sd, p + ".norm", x, 32, 1e-6)).reshape(b, c, 1, h * w)
    for d in range(depth):
        t = _tblock(sd, f"{p}.transformer_blocks.{d}", t, ctx, heads)
    return _conv(sd, p + ".proj_out", t.reshape(b, c, h, w)) + res


def _as_list(v, n):
    return list(v) if isinstance(v, (list, tuple)) else [v] * n


def unet_forward(sd, cfg, sample, timestep, encoder_hidden_states, time_ids=None, text_embeds=None,
                 additional_residuals=None):
    """Returns noise_pred (B, out_ch, H, W) fp32.  ``encoder_hidden_states`` is (B, D, 1, S)."""
    boc = list(cfg["block_out_channels"])
    nb = len(boc)
    lpb = cfg.get("layers_per_block", 2)
    heads = _as_list(cfg.get("attention_head_dim", 8), nb)
    depth = _as_list(cfg.get("transformer_layers_per_block", 1), nb)
    groups = cfg.get("norm_num_groups", 32)
    eps = cfg.get("norm_eps", 1e-5)
    down_types = cfg.get("down_block_types",
                         ("CrossAttnDownBlock2D",) * (nb - 1) + ("DownBlock2D",))
    up_types = cfg.get("up_block_types", ("UpBlock2D",) + ("CrossAttnUpBlock2D",) * (nb - 1))

    sample, ctx = _f(sample), _f(encoder_hidden_states)
    temb = _time_mlp(sd, "time_embedding",
                     timestep_embedding(timestep, boc[0], cfg.get("flip_sin_to_cos", True),
                                        cfg.get("freq_shift", 0)))
    if cfg.get("addition_embed_type") == "text_time":
        te = timestep_embedding(time_ids.flatten(), cfg["addition_time_embed_dim"],
                                cfg.get("flip_sin_to_cos", True), cfg.get("freq_shift", 0))
        te = te.reshape(text_embeds.shape[0], -1)
        temb = temb + _time_mlp(sd, "add_embedding", torch.cat([_f(text_embeds), te], dim=-1))

    x = _conv(sd, "conv_in", sample, padding=1)
    skips = [x]
    for i, typ in enumerate(down_types):
        for j in range(lpb):
            x = _resnet(sd, f"down_blocks.{i}.resnets.{j}", x, temb, groups, eps)
            if typ == "CrossAttnDownBlock2D":
                x = _spatial_transformer(sd, f"down_blocks.{i}.attentions.{j}", x, ctx, heads[i], depth[i])
            skips.append(x)
        if i != nb - 1:
            x = _conv(sd, f"down_blocks.{i}.downsamplers.0.conv", x, stride=2, padding=1)
            skips.append(x)
    if additional_residuals is not None:
        skips = [s + _f(r) for s, r in zip(skips, additional_residuals[:-1])]

    x = _resnet(sd, "mid_block.resnets.0", x, temb, groups, eps)
    x = _spatial_transformer(sd, "mid_block.attentions.0", x, ctx, heads[-1], depth[-1])
    x = _resnet(sd, "mid_block.resnets.1", x, temb, groups, eps)
    if additional_residuals is not None:
        x = x + _f(additional_residuals[-1])

    rheads, rdepth = heads[::-1], depth[::-1]
    for i, typ in enumerate(up_types):
        for j in range(lpb + 1):
            x = torch.cat([x, skips.pop()], dim=1)
            x = _resnet(sd, f"up_blocks.{i}.resnets.{j}", x, temb, groups, eps)
            if typ == "CrossAttnUpBlock2D":
                x = _spatial_transformer(sd, f"up_blocks.{i}.attentions.{j}", x, ctx, rheads[i], rdepth[i])
        if i != nb - 1:
            x = F.interpolate(x, scale_factor=2.0, mode="nearest")
            x = _conv(sd, f"up_blocks.{i}.upsamplers.0.conv", x, padding=1)

    x = F.silu(_gn(sd, "conv_norm_out", x, groups, eps))
    return _conv(sd, "conv_out", x, padding=1)


def controlnet_forward(sd, cfg, sample, timestep, encoder_hidden_states, controlnet_cond):
    """Restates ``ControlNetModel.forward`` (controlnet.py:199-250) and the conditioning embedder
    (:15-47).  Returns the list of down residuals followed by the mid residual."""
    boc = list(cfg["block_out_channels"])
    nb = len(boc)
    lpb = cfg.get("layers_per_block", 2)
    heads = _as_list(cfg.get("attention_head_dim", 8), nb)
    depth = _as_list(cfg.get("transformer_layers_per_block", 1), nb)
    groups = cfg.get("norm_num_groups", 32)
    eps = cfg.get("norm_eps", 1e-5)
    ctx = encoder_hidden_states.float()
    temb = _time_mlp(sd, "time_embedding",
                     timestep_embedding(timestep, boc[0], cfg.get("flip_sin_to_cos", True), cfg.get("freq_shift", 0)))
    ce = list(cfg.get("conditioning_embedding_out_channels", (16, 32, 96, 256)))
    e = F.silu(_conv(sd, "controlnet_cond_embedding.conv_in", controlnet_cond.float(), padding=1))
    for i in range(len(ce) - 1):
        e = F.silu(_conv(sd, f"controlnet_cond_embedding.blocks.{2 * i}", e, padding=1))
        e = F.silu(_conv(sd, f"controlnet_cond_embedding.blocks.{2 * i + 1}", e, stride=2, padding=1))
    e = _conv(sd, "controlnet_cond_embedding.conv_out", e, padding=1)
    x = _conv(sd, "conv_in", sample.float(), padding=1) + e
    skips = [x]
    for i, typ in enumerate(cfg["down_block_types"]):
        for j in range(lpb):
            x = _resnet(sd, f"down_blocks.{i}.resnets.{j}", x, temb, groups, eps)
            if typ == "CrossAttnDownBlock2D":
                x = _spatial_transformer(sd, f"down_blocks.{i}.attentions.{j}", x, ctx, heads[i], depth[i])
            skips.append(x)
        if i != nb - 1:
            x = _conv(sd, f"down_blocks.{i}.downsamplers.0.conv", x, stride=2, padding=1)
            skips.append(x)
    x = _resnet(sd, "mid_block.resnets.0", x, temb, groups, eps)
    x = _spatial_transformer(sd, "mid_block.attentions.0", x, ctx, heads[-1], 1)
    x = _resnet(sd, "mid_block.resnets.1", x, temb, groups, eps)
    outs = [_conv(sd, f"controlnet_down_blocks.{k}", s) for k, s in enumerate(skips)]
    outs.append(_conv(sd, "controlnet_mid_block", x))
    return outs


# --------------------------------------------------------------------------------------
# VAE decoder (diffusers AutoencoderKL.decoder o post_quant_conv) -- parity unpinned
# --------------------------------------------------------------------------------------
def _vae_resnet(sd, p, x):
    h = _conv(sd, p + ".conv1", F.silu(_gn(sd, p + ".norm1", x, 32, 1e-6)), padding=1)
    h = _conv(sd, p + ".conv2", F.silu(_gn(sd, p + ".norm2", h, 32, 1e-6)), padding=1)
    if (p + ".conv_shortcut.weight") in sd:
        x = _conv(sd, p + ".conv_shortcut", x)
    return x + h


def _vae_attn(sd, p, x):
    b, c, h, w = x.shape
    t = _gn(sd, p + ".group_norm", x, 32, 1e-6).reshape(b, c, 1, h * w)
    q, k, v = (_conv(sd, f"{p}.to_{n}", t) for n in "qkv")
    o = attention(q, k, v, 1, c)
    return _conv(sd, p + ".to_out.0", o).reshape(b, c, h, w) + x


def vae_decode(sd, cfg, z):
    """image = decoder(post_quant_conv(z)); the 1/scaling_factor is applied by the caller
    (reference ``pipeline.py:313-320``)."""
    boc = list(cfg.get("block_out_channels", (128, 256, 512, 512)))
    lpb = cfg.get("layers_per_block", 2)
    x = _conv(sd, "post_quant_conv", z.float())
    x = _conv(sd, "decoder.conv_in", x, padding=1)
    x = _vae_resnet(sd, "decoder.mid_block.resnets.0", x)
    x = _vae_attn(sd, "decoder.mid_block.attentions.0", x)
    x = _vae_resnet(sd, "decoder.mid_block.resnets.1", x)
    for i in range(len(boc)):
        for j in range(lpb + 1):
            x = _vae_resnet(sd, f"decoder.up_blocks.{i}.resnets.{j}", x)
        if i != len(boc) - 1:
            x = F.interpolate(x, scale_factor=2.0, mode="nearest")
            x = _conv(sd, f"decoder.up_blocks.{i}.upsamplers.0.conv", x, padding=1)
    x = F.silu(_gn(sd, "decoder.conv_norm_out", x, 32, 1e-6))
    return _conv(sd, "decoder.conv_out", x, padding=1)


def vae_encode(sd, cfg, x):
    """moments = quant_conv(encoder(x)) (torch2coreml.py:739-749); x in [-1, 1], (B, 3, H, W) ->
    (B, 2 * latent_channels, H/8, W/8).  diffusers Encoder: conv_in, DownEncoderBlock2D x N (ResNets, then
    Downsample2D(padding=0): F.pad(x, (0, 1, 0, 1)) + 3x3 stride-2 conv), mid block, GroupNorm + SiLU, conv_out.
    parity unpinned (diffusers is not installed; same status as vae_decode)."""
    boc = list(cfg.get("block_out_channels", (128, 256, 512, 512)))
    lpb = cfg.get("layers_per_block", 2)
    h = _conv(sd, "encoder.conv_in", x.float(), padding=1)
    for i in range(len(boc)):
        for j in range(lpb):
            h = _vae_resnet(sd, f"encoder.down_blocks.{i}.resnets.{j}", h)
        if i != len(boc) - 1:
            h = _conv(sd, f"encoder.down_blocks.{i}.downsamplers.0.conv", F.pad(h, (0, 1, 0, 1)), stride=2)
    h = _vae_resnet(sd, "encoder.mid_block.resnets.0", h)
    h = _vae_attn(sd, "encoder.mid_block.attentions.0", h)
    h = _vae_resnet(sd, "encoder.mid_block.resnets.1", h)
    h = F.silu(_gn(sd, "encoder.conv_norm_out", h, 32, 1e-6))
    return _conv(sd, "quant_conv", _conv(sd, "encoder.conv_out", h, padding=1))


def sample_latents(moments, noise, scaling_factor=0.18215):
    """DiagonalGaussianDistribution.sample (Encoder.swift: mean + exp(0.5 * clamp(logvar, -30, 20)) * noise),
    times the scaling factor."""
    mean, logvar = moments.chunk(2, dim=1)
    return (mean + torch.exp(0.5 * logvar.clamp(-30.0, 20.0)) * noise) * scaling_factor


def postprocess_image(img):
    """pipeline.py:317-318: clip(x/2+0.5, 0, 1), NCHW -> NHWC."""
    return (img / 2 + 0.5).clamp(0, 1).permute(0, 2, 3, 1)


# --------------------------------------------------------------------------------------
# Schedulers (diffusers 0.30.2 semantics; Swift twins cited) -- parity unpinned
# --------------------------------------------------------------------------------------
def alphas_cumprod(beta_start=0.00085, beta_end=0.012, n=1000):
    """scaled_linear betas (Scheduler.swift:175-186)."""
    betas = torch.linspace(beta_start ** 0.5, beta_end ** 0.5, n, dtype=torch.float32) ** 2
    return torch.cumprod(1.0 - betas, dim=0)


def leading_timesteps(num_steps, n_train=1000, steps_offset=1):
    """'leading' spacing (Scheduler.swift:187-191): 20 steps -> 951, 901, ..., 1."""
    ratio = n_train // num_steps
    return [int(round(i * ratio)) + steps_offset for i in range(num_steps)][::-1]


def cfg_combine(eps_uncond, eps_text, guidance_scale):
    """pipeline.py:559-562 / StableDiffusionPipeline.swift:469-483."""
    return eps_uncond + guidance_scale * (eps_text - eps_uncond)


def ddim_step(eps, t, x, abar, num_steps, n_train=1000):
    """DDIM eta=0, epsilon prediction, set_alpha_to_one=False (SURVEY Appendix B2);
    equals DPM-Solver++ first-order update (DPMSolverMultistepScheduler.swift:153-174)."""
    t_prev = t - n_train // num_steps
    a_t = abar[t]
    a_p = abar[t_prev] if t_prev >= 0 else abar[0]
    x0 = (x - (1 - a_t).sqrt() * eps) / a_t.sqrt()
    return a_p.sqrt() * x0 + (1 - a_p).sqrt() * eps


class DPMSolverPP2M:
    """DPM-Solver++(2M), midpoint, epsilon prediction, linspace spacing, lower_order_final
    when < 15 steps (DPMSolverMultistepScheduler.swift:61-126, :135-151, :156-244)."""

    def __init__(self, num_steps, abar=None, n_train=1000, final_sigmas_type="sigma_min"):
        self.abar = alphas_cumprod() if abar is None else abar
        self.n = num_steps
        self.final_sigmas_type = final_sigmas_type  # "zero": diffusers 0.30.2 default (last step -> x0)
        ts = torch.linspace(0, n_train - 1, num_steps + 1).round().long().flip(0)[:-1]
        self.timesteps = [int(t) for t in ts]
        self.alpha = self.abar.sqrt()
        self.sigma = (1 - self.abar).sqrt()
        self.lam = self.alpha.log() - self.sigma.log()
        self.x0_hist = []
        self.lower_order_nums = 0
        self.lower_order_final = num_steps < 15

    def _prev_t(self, i):
        return self.timesteps[i + 1] if i + 1 < self.n else 0

    def step(self, eps, i, x):
        t = self.timesteps[i]
        p = self._prev_t(i)
        x0 = (x - self.sigma[t] * eps) / self.alpha[t]
        self.x0_hist.append(x0)
        self.x0_hist = self.x0_hist[-2:]
        lower_final = (i == self.n - 1) and self.lower_order_final
        lower_second = (i == self.n - 2) and self.lower_order_final  # Swift :221-222
        order1 = self.lower_order_nums < 1 or lower_final or lower_second
        h = self.lam[p] - self.lam[t]
        if i == self.n - 1 and self.final_sigmas_type == "zero":
            out = x0
        elif order1:
            out = (self.sigma[p] / self.sigma[t]) * x - self.alpha[p] * (torch.exp(-h) - 1.0) * x0
        else:
            t1 = self.timesteps[i - 1]
            h0 = self.lam[t] - self.lam[t1]
            r0 = h0 / h
            d0 = self.x0_hist[-1]
            d1 = (1.0 / r0) * (self.x0_hist[-1] - self.x0_hist[-2])
            em1 = torch.exp(-h) - 1.0
            out = (self.sigma[p] / self.sigma[t]) * x - self.alpha[p] * em1 * d0 \
                - 0.5 * self.alpha[p] * em1 * d1
        if self.lower_order_nums < 2:
            self.lower_order_nums += 1
        return out


class PNDM:
    """PLMS (skip_prk_steps=True) epsilon prediction (Scheduler.swift:137-344)."""

    def __init__(self, num_steps, abar=None, n_train=1000, steps_offset=1):
        self.abar = alphas_cumprod() if abar is None else abar
        self.n_train = n_train
        self.num_steps = num_steps
        ratio = n_train // num_steps
        base = [int(round(i * ratio)) + steps_offset for i in range(num_steps)]
        # duplicated second-to-last element (Scheduler.swift:197-201)
        ts = base[:-1] + base[-2:-1] + base[-1:]
        self.timesteps = ts[::-1]
        self.ets = []
        self.counter = 0
        self.cur_sample = None

    def _prev_sample(self, x, t, t_prev, eps):
        a_t = self.abar[t]
        a_p = self.abar[t_prev] if t_prev >= 0 else self.abar[0]
        b_t, b_p = 1 - a_t, 1 - a_p
        coeff = (a_p / a_t).sqrt()
        denom = a_t * b_p.sqrt() + (a_t * b_t * a_p).sqrt()
        return coeff * x - (a_p - a_t) * eps / denom

    def step(self, eps, t, x):
        ratio = self.n_train // self.num_steps
        t_prev = t - ratio
        if self.counter != 1:
            self.ets = self.ets[-3:]
            self.ets.append(eps)
        else:
            t_prev = t
            t = t + ratio
        if len(self.ets) == 1 and self.counter == 0:
            e = eps
            self.cur_sample = x
        elif len(self.ets) == 1 and self.counter == 1:
            e = (eps + self.ets[-1]) / 2
            x = self.cur_sample
            self.cur_sample = None
        elif len(self.ets) == 2:
            e = (3 * self.ets[-1] - self.ets[-2]) / 2
        elif len(self.ets) == 3:
            e = (23 * self.ets[-1] - 16 * self.ets[-2] + 5 * self.ets[-3]) / 12
        else:
            e = (55 * self.ets[-1] - 59 * self.ets[-2] + 37 * self.ets[-3] - 9 * self.ets[-4]) / 24
        self.counter += 1
        return self._prev_sample(x, t, t_prev, e)


def compute_psnr(a, b):
    """Restates ``torch2coreml.py:59-74``: 20 log10(max|b| / rmse(a-b)), eps-guarded."""
    a = a.double().flatten()
    b = b.double().flatten()
    eps = 1e-5
    eps2 = 1e-10
    mse = ((a - b) ** 2).mean()
    return float(20 * torch.log10((b.abs().max() + eps) / (mse.sqrt() + eps2)))
