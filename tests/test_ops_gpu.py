"""GPU parity tests of the individual C-ABI ops against plain PyTorch fp32 references of the same
op (inputs rounded to fp16 first, so the only differences are accumulation order and the fp16
rounding of the stored result).  All calls go through ``libb200sd.so``."""
import math

import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu


def _close(got, ref, atol, rtol, what):
    got = got.float()
    ref = ref.float()
    err = (got - ref).abs()
    tol = atol + rtol * ref.abs()
    bad = err > tol
    if bad.any():
        idx = torch.nonzero(bad)[0].tolist()
        raise AssertionError(f"{what}: {int(bad.sum())}/{bad.numel()} mismatches, max err {err.max().item():.4g} "
                             f"(ref absmax {ref.abs().max().item():.4g}) first at {idx}: got "
                             f"{got[tuple(idx)].item():.5g} ref {ref[tuple(idx)].item():.5g}")


def _rand(*shape, scale=1.0, seed=0):
    g = torch.Generator(device="cuda").manual_seed(seed)
    return (torch.randn(*shape, generator=g, device="cuda") * scale).half()


@pytest.mark.parametrize("m,n,k", [(128, 64, 64), (256, 128, 64), (128, 256, 256), (8192, 320, 320),
                                   (154, 320, 1024), (2048, 640, 640), (512, 1280, 5120), (100, 48, 96)])
def test_linear_plain(cuda_lib, m, n, k):
    x, w = _rand(m, k, seed=1), _rand(n, k, scale=k ** -0.5, seed=2)
    out = cuda_lib.linear(x, w)
    torch.cuda.synchronize()
    _close(out, x.float() @ w.float().t(), 2e-3, 2e-3, f"linear {m}x{n}x{k}")


def test_linear_bias_residual_f32(cuda_lib):
    m, n, k = 2048, 640, 640
    x, w, r = _rand(m, k, seed=1), _rand(n, k, scale=k ** -0.5, seed=2), _rand(m, n, seed=3)
    b = torch.randn(n, device="cuda")
    ref = x.float() @ w.float().t() + b + r.float()
    _close(cuda_lib.linear(x, w, b, r), ref, 3e-3, 2e-3, "linear+bias+res fp16")
    _close(cuda_lib.linear(x, w, b, r, out_dtype=torch.float32), ref, 1e-3, 1e-3, "linear+bias+res fp32")


def test_linear_geglu(cuda_lib):
    m, c = 512, 320
    x, w = _rand(m, c, seed=1), _rand(8 * c, c, scale=c ** -0.5, seed=2)
    b = torch.randn(8 * c, device="cuda")
    y = x.float() @ w.float().t() + b
    a, g = y.chunk(2, dim=1)
    ref = a * F.gelu(g)
    # engine layout: rows interleaved (value_i, gate_i)
    wi = torch.stack([w[: 4 * c], w[4 * c:]], dim=1).reshape(8 * c, c).contiguous()
    bi = torch.stack([b[: 4 * c], b[4 * c:]], dim=1).reshape(8 * c).contiguous()
    _close(cuda_lib.linear(x, wi, bi, geglu=True), ref, 3e-3, 3e-3, "geglu")


def test_linear_two_sources(cuda_lib):
    m, n, c0, c1 = 512, 320, 640, 320
    x0, x1 = _rand(m, c0, seed=1), _rand(m, c1, seed=2)
    w = _rand(n, c0 + c1, scale=(c0 + c1) ** -0.5, seed=3)
    ref = torch.cat([x0, x1], 1).float() @ w.float().t()
    _close(cuda_lib.linear(x0, w, x1=x1), ref, 2e-3, 2e-3, "two-source linear")


@pytest.mark.parametrize("split", [2, 4, 7])
def test_linear_split_k(cuda_lib, split):
    m, n, k = 128, 1280, 1280
    x, w, r = _rand(m, k, seed=1), _rand(n, k, scale=k ** -0.5, seed=2), _rand(m, n, seed=3)
    b = torch.randn(n, device="cuda")
    ref = x.float() @ w.float().t() + b + r.float()
    _close(cuda_lib.linear(x, w, b, r, split_k=split), ref, 3e-3, 2e-3, f"split-K {split}")


def _conv_ref(x, w, b=None, stride=1):
    y = F.conv2d(x.float().permute(0, 3, 1, 2), w.float(), None if b is None else b.float(), stride=stride, padding=1)
    return y.permute(0, 2, 3, 1).contiguous()


def _pack(w):  # [Co, Ci, 3, 3] -> [Co, 9*Ci] with k = (ky*3+kx)*Ci + c
    return w.permute(0, 2, 3, 1).reshape(w.shape[0], -1).contiguous()


@pytest.mark.parametrize("n,h,w,ci,co", [(2, 64, 64, 64, 64), (2, 16, 16, 128, 128), (2, 32, 32, 320, 640),
                                         (2, 8, 8, 1280, 1280), (1, 64, 64, 320, 320), (2, 4, 4, 128, 128),
                                         (1, 24, 24, 64, 96)])
def test_conv3x3(cuda_lib, n, h, w, ci, co):
    x = _rand(n, h, w, ci, seed=1)
    wt = _rand(co, ci, 3, 3, scale=(9 * ci) ** -0.5, seed=2)
    b = torch.randn(co, device="cuda")
    out = cuda_lib.conv3x3(x, _pack(wt), b)
    torch.cuda.synchronize()
    _close(out, _conv_ref(x, wt, b), 3e-3, 3e-3, f"conv3x3 {n}x{h}x{w} {ci}->{co}")


@pytest.mark.parametrize("m,split,out_dtype", [(128, 8, torch.float16), (200, 4, torch.float16), (512, 2, torch.float32)])
def test_linear_split_k_cluster(cuda_lib, m, split, out_dtype):
    """split-K reduced inside a thread-block cluster through DSMEM (2 / 4 / 8 CTAs per tile), ragged last tile."""
    n, k = 640, 2560
    x, w, r = _rand(m, k, seed=1), _rand(n, k, scale=k ** -0.5, seed=2), _rand(m, n, seed=3)
    b = torch.randn(n, device="cuda")
    ref = x.float() @ w.float().t() + b + r.float()
    plan = cuda_lib.describe_plan(0, m=m, n=n, c0=k, has_residual=True, split_k=split)
    assert "cluster=1" in plan and f"splits={split} " in plan, plan
    out = cuda_lib.linear(x, w, b, r, split_k=split, out_dtype=out_dtype)
    _close(out, ref, 3e-3, 2e-3, f"cluster split-K {split}")
    # bitwise reproducible: fixed rank order of the DSMEM reduction
    assert torch.equal(out, cuda_lib.linear(x, w, b, r, split_k=split, out_dtype=out_dtype))


def test_conv3x3_split_k_cluster_temb_residual(cuda_lib):
    n, h, w, c0, c1, co = 2, 16, 16, 640, 320, 640
    x0, x1 = _rand(n, h, w, c0, seed=1), _rand(n, h, w, c1, seed=2)
    wt = _rand(co, c0 + c1, 3, 3, scale=(9 * (c0 + c1)) ** -0.5, seed=3)
    bias_img = torch.randn(n, co, device="cuda")
    res = _rand(n, h, w, co, seed=4)
    ref = _conv_ref(torch.cat([x0, x1], -1), wt) + bias_img[:, None, None, :] + res.float()
    for split in (4, 8):
        out = cuda_lib.conv3x3(x0, _pack(wt), bias_img, res, x1=x1, bias_rows=h * w, split_k=split)
        _close(out, ref, 4e-3, 3e-3, f"conv cluster split-K {split}")


def test_conv3x3_small_channels(cuda_lib):
    # conv_in: 4 channels padded to 8; conv_out: 4 output channels, fp32 out
    x = _rand(2, 64, 64, 8, seed=1)
    x[..., 4:] = 0
    wt = _rand(320, 8, 3, 3, scale=36 ** -0.5, seed=2)
    _close(cuda_lib.conv3x3(x, _pack(wt)), _conv_ref(x, wt), 3e-3, 3e-3, "conv_in")
    x2 = _rand(2, 64, 64, 320, seed=3)
    w2 = _rand(4, 320, 3, 3, scale=2880 ** -0.5, seed=4)
    b2 = torch.randn(4, device="cuda")
    _close(cuda_lib.conv3x3(x2, _pack(w2), b2, out_dtype=torch.float32), _conv_ref(x2, w2, b2), 2e-3, 2e-3, "conv_out")


def test_conv3x3_temb_residual_two_sources(cuda_lib):
    n, h, w, c0, c1, co = 2, 16, 16, 128, 64, 128
    x0, x1 = _rand(n, h, w, c0, seed=1), _rand(n, h, w, c1, seed=2)
    wt = _rand(co, c0 + c1, 3, 3, scale=(9 * (c0 + c1)) ** -0.5, seed=3)
    bias_img = torch.randn(n, co, device="cuda")  # conv bias + per-image time embedding
    res = _rand(n, h, w, co, seed=4)
    ref = _conv_ref(torch.cat([x0, x1], -1), wt) + bias_img[:, None, None, :] + res.float()
    out = cuda_lib.conv3x3(x0, _pack(wt), bias_img, res, x1=x1, bias_rows=h * w)
    _close(out, ref, 4e-3, 3e-3, "conv temb+res+2src")


@pytest.mark.parametrize("n,h,w,c", [(2, 64, 64, 320), (2, 16, 16, 128), (2, 8, 8, 64)])
def test_conv3x3_stride2(cuda_lib, n, h, w, c):
    x = _rand(n, h, w, c, seed=1)
    wt = _rand(c, c, 3, 3, scale=(9 * c) ** -0.5, seed=2)
    b = torch.randn(c, device="cuda")
    _close(cuda_lib.conv3x3(x, _pack(wt), b, stride=2), _conv_ref(x, wt, b, stride=2), 3e-3, 3e-3, "conv s2")


@pytest.mark.parametrize("n,h,w,c", [(1, 64, 64, 64), (2, 16, 16, 128), (1, 24, 40, 64)])
def test_conv3x3_stride2_pad_after_only(cuda_lib, n, h, w, c):
    """diffusers Downsample2D(padding=0): F.pad(x, (0, 1, 0, 1)) then a 3x3 stride-2 convolution (VAE encoder)."""
    x = _rand(n, h, w, c, seed=1)
    wt = _rand(c, c, 3, 3, scale=(9 * c) ** -0.5, seed=2)
    b = torch.randn(c, device="cuda")
    ref = F.conv2d(F.pad(x.float().permute(0, 3, 1, 2), (0, 1, 0, 1)), wt.float(), b, stride=2).permute(0, 2, 3, 1)
    out = cuda_lib.conv3x3(x, _pack(wt), b, stride=2, pad_after_only=True)
    assert out.shape == ref.shape
    _close(out, ref.contiguous(), 3e-3, 3e-3, "conv s2 pad-after-only")


@pytest.mark.parametrize("n,hw,c0,c1,silu", [(2, 64, 320, 0, True), (2, 32, 640, 0, False), (2, 16, 1280, 640, True),
                                             (2, 8, 64, 0, True), (1, 64, 128, 128, False)])
def test_group_norm(cuda_lib, n, hw, c0, c1, silu):
    x0 = _rand(n, hw, hw, c0, seed=1) + 0.5
    x1 = _rand(n, hw, hw, c1, scale=2.0, seed=2) if c1 else None
    c = c0 + c1
    g, b = torch.randn(c, device="cuda"), torch.randn(c, device="cuda")
    xc = x0 if x1 is None else torch.cat([x0, x1], -1)
    ref = F.group_norm(xc.float().permute(0, 3, 1, 2), 32, g, b, 1e-5)
    if silu:
        ref = F.silu(ref)
    out = cuda_lib.group_norm(x0, g, b, 32, 1e-5, silu=silu, x1=x1)
    _close(out, ref.permute(0, 2, 3, 1), 4e-3, 2e-3, "group_norm")


@pytest.mark.parametrize("rows,c", [(8192, 320), (2048, 640), (512, 1280), (77, 64), (100, 2048)])
def test_layer_norm(cuda_lib, rows, c):
    x = _rand(rows, c, seed=1) * 2 + 0.3
    g, b = torch.randn(c, device="cuda"), torch.randn(c, device="cuda")
    _close(cuda_lib.layer_norm(x, g, b), F.layer_norm(x.float(), (c,), g, b, 1e-5), 4e-3, 2e-3, "layer_norm")


def _attn_ref(q, k, v, batch, heads, sq, sk, mask=None):
    d = 64
    qh = q.float().reshape(batch, sq, heads, d).permute(0, 2, 1, 3)
    kh = k.float().reshape(batch, sk, heads, d).permute(0, 2, 1, 3)
    vh = v.float().reshape(batch, sk, heads, d).permute(0, 2, 1, 3)
    s = qh @ kh.transpose(-1, -2) * d ** -0.5
    if mask is not None:
        s = s + mask[:, None, None, :]
    return (s.softmax(-1) @ vh).permute(0, 2, 1, 3).reshape(batch * sq, heads * d)


@pytest.mark.parametrize("batch,heads,sq,sk", [(1, 1, 128, 128), (2, 2, 256, 256), (2, 5, 1024, 1024), (2, 5, 256, 77),
                                               (2, 20, 64, 64), (1, 3, 200, 333), (2, 5, 4096, 4096)])
def test_attention(cuda_lib, batch, heads, sq, sk):
    c = heads * 64
    q, k, v = _rand(batch * sq, c, seed=1), _rand(batch * sk, c, seed=2), _rand(batch * sk, c, seed=3)
    out = cuda_lib.attention(q, k, v, batch, heads, sq, sk)
    torch.cuda.synchronize()
    _close(out, _attn_ref(q, k, v, batch, heads, sq, sk), 3e-3, 3e-3, f"attention {batch}x{heads}x{sq}x{sk}")


@pytest.mark.parametrize("batch,heads,s", [(2, 2, 77), (1, 3, 300), (2, 16, 128)])
def test_attention_causal(cuda_lib, batch, heads, s):
    """Causal mask of the CLIP text encoder (key j visible to query i iff j <= i), incl. halves above the diagonal
    that are skipped and the diagonal halves that take the predicated path."""
    c = heads * 64
    q, k, v = _rand(batch * s, c, seed=1), _rand(batch * s, c, seed=2), _rand(batch * s, c, seed=3)
    qh, kh, vh = (t.float().view(batch, s, heads, 64).transpose(1, 2) for t in (q, k, v))
    sc = qh @ kh.transpose(-1, -2) * 64 ** -0.5 + torch.full((s, s), float("-inf"), device="cuda").triu(1)
    ref = (torch.softmax(sc, -1) @ vh).transpose(1, 2).reshape(batch * s, c)
    _close(cuda_lib.attention(q, k, v, batch, heads, s, s, causal=True), ref, 3e-3, 3e-3, f"causal attention {s}")


def test_text_encoder_ops(cuda_lib):
    ids = torch.randint(0, 500, (2, 77), device="cuda").float()
    tok, pos = _rand(500, 128, seed=1), _rand(77, 128, seed=2)
    ref = (tok[ids.long()] + pos[None]).reshape(2 * 77, 128).float()
    _close(cuda_lib.embed_tokens(ids, tok, pos), ref, 1e-3, 2e-3, "embed_tokens")
    x, w = _rand(154, 256, seed=3), _rand(512, 256, scale=256 ** -0.5, seed=4)
    b = torch.randn(512, device="cuda")
    y = x.float() @ w.float().t() + b
    _close(cuda_lib.linear(x, w, b, act=2), F.gelu(y), 3e-3, 3e-3, "linear + GELU")
    _close(cuda_lib.linear(x, w, b, act=3), y * torch.sigmoid(1.702 * y), 3e-3, 3e-3, "linear + quick-GELU")


def test_attention_fused_qkv_and_mask(cuda_lib):
    batch, heads, s = 2, 5, 256
    c = heads * 64
    qkv = _rand(batch * s, 3 * c, seed=1)
    q, k, v = qkv[:, :c], qkv[:, c:2 * c], qkv[:, 2 * c:]
    out = cuda_lib.attention(q, k, v, batch, heads, s, s)
    _close(out, _attn_ref(q, k, v, batch, heads, s, s), 3e-3, 3e-3, "attention fused-qkv views")
    mask = torch.zeros(batch, s, device="cuda")
    mask[:, 100:] = -1e4  # the reference's additive mask convention (unet.py:99-114)
    out = cuda_lib.attention(q, k, v, batch, heads, s, s, mask=mask)
    _close(out, _attn_ref(q, k, v, batch, heads, s, s, mask), 3e-3, 3e-3, "attention mask")


def test_small_kernels(cuda_lib):
    lib = cuda_lib
    x = torch.randn(2, 4, 16, 16, device="cuda")
    nhwc = lib.nchw_to_nhwc(x, c_pad=8)
    assert torch.equal(nhwc[..., :4], x.permute(0, 2, 3, 1).half()) and (nhwc[..., 4:] == 0).all()
    back = lib.nhwc_to_nchw_f32(nhwc, c=4)
    assert torch.equal(back, x.half().float())
    y = _rand(2, 8, 8, 64, seed=5)
    up = lib.upsample2x(y)
    assert torch.equal(up, y.repeat_interleave(2, 1).repeat_interleave(2, 2))
    a, b = _rand(1000, 64, seed=6), _rand(1000, 64, seed=7)
    _close(lib.add(a, b), a.float() + b.float(), 1e-3, 1e-3, "add")
    ctx = torch.randn(2, 96, 1, 77, device="cuda")
    tok = lib.ctx_to_tokens(ctx)
    assert torch.equal(tok, ctx[:, :, 0, :].permute(0, 2, 1).reshape(2 * 77, 96).half())
    t = torch.tensor([981.0, 1.0], device="cuda")
    emb = lib.timestep_embedding(t, 320)
    half = 160
    fr = torch.exp(-math.log(10000) * torch.arange(half, device="cuda", dtype=torch.float32) / half)
    ang = t[:, None] * fr[None]
    _close(emb, torch.cat([ang.cos(), ang.sin()], -1), 2e-4, 1e-4, "timestep embedding")
    xs = torch.randn(2, 320, device="cuda")
    w = _rand(1280, 320, scale=320 ** -0.5, seed=8)
    bb = torch.randn(1280, device="cuda")
    _close(lib.linear_small(xs, w, bb, act_out=True), F.silu(xs @ w.float().t() + bb), 1e-3, 1e-3, "linear_small")
    _close(lib.linear_small(xs, w, bb, add=bb, act_in=True), F.silu(xs) @ w.float().t() + 2 * bb, 1e-3, 1e-3,
           "linear_small act_in")
    img = torch.randn(1, 8, 8, 8, device="cuda").half()
    pf, pu = lib.image_postprocess(img, c=3, want_u8=True)
    ref = (img[..., :3].float() / 2 + 0.5).clamp(0, 1)
    _close(pf, ref, 1e-6, 0, "image post f32")
    assert (pu.float() - ref * 255).abs().max() <= 0.5 + 1e-3


def test_cfg_scheduler_step(cuda_lib):
    lib = cuda_lib
    n, c, h, w = 2, 4, 16, 16
    eps = torch.randn(2 * n, c, h, w, device="cuda")
    x = torch.randn(n, c, h, w, device="cuda")
    hist = torch.randn(4, n, c, h, w, device="cuda")
    k = lib.StepCoeffs()
    k.guidance, k.cx, k.ce = 7.5, 0.9, -0.2
    k.ch[0], k.ch[1] = 0.3, -0.1
    k.x0_cx, k.x0_ce = 1.1, -0.4
    k.n_hist, k.push_eps_slot, k.push_x0_slot, k.push_x_slot = 2, -1, 3, 2
    e = eps[:n] + 7.5 * (eps[n:] - eps[:n])
    ref = 0.9 * x - 0.2 * e + 0.3 * hist[0] - 0.1 * hist[1]
    ref_x0 = 1.1 * x - 0.4 * e
    lat = x.clone()
    den = torch.empty_like(x)
    unet_in = torch.zeros(2 * n, h, w, 8, device="cuda", dtype=torch.float16)
    hist2 = hist.clone()
    lib.cfg_scheduler_step(eps, lat, k, hist=hist2, denoised=den, unet_in=unet_in)
    _close(lat, ref, 1e-5, 1e-5, "step latents")
    _close(den, ref_x0, 1e-5, 1e-5, "step x0")
    _close(hist2[3], ref_x0, 1e-5, 1e-5, "history push")
    assert torch.equal(hist2[:2], hist[:2]) and torch.equal(hist2[2], x)
    want = ref.permute(0, 2, 3, 1)  # fp16 rounding of an FMA-contracted fp32 value: compare to 1 half-ulp
    _close(unet_in[:n, ..., :4], want, 2e-3, 1e-3, "next unet input (uncond half)")
    _close(unet_in[n:, ..., :4], want, 2e-3, 1e-3, "next unet input (cond half)")
    assert (unet_in[..., 4:] == 0).all()


def test_attention_large_scores_take_the_rescale_path(cuda_lib):
    """Scores whose running maximum grows by orders of magnitude from one 64-key half to the next force large rescales of
    the running output O (attention.cu online softmax); random-init inputs almost never do."""
    b, h, s, d = 1, 2, 512, 64
    g = torch.Generator(device="cuda").manual_seed(5)
    q = torch.randn(b * s, h * d, generator=g, device="cuda")
    k = torch.randn(b * s, h * d, generator=g, device="cuda")
    v = torch.randn(b * s, h * d, generator=g, device="cuda")
    # later keys are scaled up so that every half raises the row maxima by a large step
    ramp = torch.linspace(0.5, 12.0, s, device="cuda").repeat(b)[:, None]
    k = (k * ramp).half()
    q, v = (q * 3.0).half(), v.half()
    out = cuda_lib.attention(q, k, v, b, h, s, s)
    qf, kf, vf = (t.float().reshape(b, s, h, d).permute(0, 2, 1, 3) for t in (q, k, v))
    ref = torch.softmax(qf @ kf.transpose(-1, -2) * d ** -0.5, dim=-1) @ vf
    ref = ref.permute(0, 2, 1, 3).reshape(b * s, h * d)
    _close(out, ref, 3e-3, 3e-3, "attention with growing score maxima")


@pytest.mark.parametrize("batch,heads,sq,sk,masked", [(2, 5, 4096, 4096, False), (1, 5, 4096, 4096, False),
                                                      (2, 10, 2304, 2304, False), (2, 5, 4000, 3970, False),
                                                      (1, 5, 4096, 2048, True)])
def test_attention_stream_k(cuda_lib, monkeypatch, batch, heads, sq, sk, masked):
    """Shapes whose query tiles fill the 296 CTA slots badly are cut into equal (query tile x K/V tile) ranges per CTA
    (attention.cu `attention_slots`); the pieces of a split tile are merged in a fixed order, so the result matches the
    one-CTA-per-tile schedule to rounding, is bit-reproducible, and leaves the workspace counters at zero."""
    c = heads * 64
    q, k, v = _rand(batch * sq, c, seed=1), _rand(batch * sk, c, seed=2), _rand(batch * sk, c, seed=3)
    # growing keys: pieces of one tile end with very different reference maxima, so the merge has to rescale
    k = (k.float() * torch.linspace(0.5, 6.0, sk, device="cuda").repeat(batch)[:, None]).half()
    mask = None
    if masked:
        mask = torch.zeros(batch, sk, device="cuda")
        mask[:, ::3] = -1e4
    ref = _attn_ref(q, k, v, batch, heads, sq, sk, mask)
    out = cuda_lib.attention(q, k, v, batch, heads, sq, sk, mask=mask)
    _close(out, ref, 3e-3, 3e-3, f"stream-K attention {batch}x{heads}x{sq}x{sk}")
    for _ in range(3):
        assert torch.equal(out, cuda_lib.attention(q, k, v, batch, heads, sq, sk, mask=mask))
    counters = cuda_lib._attention_workspace(q.device)[:65536]
    assert int(counters.max()) == 0
    monkeypatch.setenv("B200SD_ATTN_STREAMK", "0")
    whole = cuda_lib.attention(q, k, v, batch, heads, sq, sk, mask=mask)
    monkeypatch.delenv("B200SD_ATTN_STREAMK")
    _close(whole, ref, 3e-3, 3e-3, "one CTA per query tile")
    assert (out.float() - whole.float()).abs().max().item() <= 2e-3
