"""CPU rehearsal of the per-launch checks of test_op_launches_gpu.py: every bound in op_refs.py accepts an fp32
emulation of its kernel and rejects each perturbed reference; and the wrappers whose kernels take a single fp16 / fp32
type flag refuse every other input type before any launch."""
import os
import sys

import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import op_refs as OR  # noqa: E402

F16, BF16 = torch.float16, torch.bfloat16


def _gn_input(g, n, hw, c, groups, rho, dt):
    off = rho * torch.randn(groups, generator=g).sign().repeat_interleave(c // groups)
    ramp = torch.linspace(-1.0, 1.0, hw)[None, :, None]
    return (torch.randn(n, hw, c, generator=g) + off + ramp).to(dt)


def _gn_emulated(x, gamma, beta, groups, eps, silu, dt):
    """fp32 one-pass statistics (sum and sum of squares), as the kernels take them."""
    n, hw, c = x.shape
    xf = x.float().reshape(n, hw, groups, c // groups)
    cnt = hw * (c // groups)
    mean = xf.sum(dim=(1, 3)) / cnt
    var = torch.clamp((xf * xf).sum(dim=(1, 3)) / cnt - mean * mean, min=0)
    y = (xf - mean[:, None, :, None]) * torch.rsqrt(var + eps)[:, None, :, None]
    y = y.reshape(n, hw, c) * gamma + beta
    return (y * torch.sigmoid(y) if silu else y).to(dt)


@pytest.mark.parametrize("dt", [F16, BF16])
@pytest.mark.parametrize("rho", [0.0, 10.0, 30.0])
@pytest.mark.parametrize("silu", [False, True])
def test_group_norm_bound(dt, rho, silu):
    g = torch.Generator().manual_seed(1)
    n, hw, c, groups = 2, 256, 64, 8
    x = _gn_input(g, n, hw, c, groups, rho, dt)
    gamma, beta = 1 + 0.2 * torch.randn(c, generator=g), 0.1 * torch.randn(c, generator=g)
    xd = x.double()
    ref, tol = OR.group_norm(xd, gamma, beta, groups, 1e-5, silu, dt)
    assert OR.worst(_gn_emulated(x, gamma, beta, groups, 1e-5, silu, dt), ref, tol) <= 1.0
    for stats in (OR.gn_stats(xd, groups, shift=8), OR.gn_stats(xd, groups, px=slice(0, hw - hw // 8))):
        alt = OR.group_norm(xd, gamma, beta, groups, 1e-5, silu, dt, stats=stats)[0]
        assert OR.rejects(alt, ref, tol)


def test_layer_norm_bound():
    g = torch.Generator().manual_seed(2)
    x = (100 + torch.randn(9, 520, generator=g)).half()
    gamma, beta = 1 + 0.2 * torch.randn(520, generator=g), 0.1 * torch.randn(520, generator=g)
    ref, tol = OR.layer_norm(x.double(), gamma, beta, 1e-5)
    xf = x.float()
    mu = xf.mean(-1, keepdim=True)
    emu = ((xf - mu) * torch.rsqrt(((xf - mu) ** 2).mean(-1, keepdim=True) + 1e-5) * gamma + beta).half()
    assert OR.worst(emu, ref, tol) <= 1.0
    assert OR.rejects(OR.layer_norm(x.double(), gamma, beta, 1e-5, shift=8)[0], ref, tol)


@pytest.mark.parametrize("dt", [F16, BF16])
def test_softmax_bound(dt):
    g = torch.Generator().manual_seed(3)
    s = torch.randn(6, 257, generator=g)
    s[1, 5] = 60.0
    for scale in (1e-6, 0.125, 300.0):
        ref, tol = OR.softmax_rows(s, scale, dt)
        z = s * (torch.tensor(scale) * torch.tensor(1.4426950408889634))
        e = torch.exp2(z - z.max(-1, keepdim=True).values)
        emu = (e * (1.0 / e.sum(-1, keepdim=True))).to(dt)
        assert OR.worst(emu, ref, tol) <= 1.0
        if scale < 1:  # at scale 300 every row is one-hot: the last column holds nothing to miss
            assert OR.rejects(OR.softmax_rows(s, scale, dt, drop_last=True)[0], ref, tol)


def test_linear_small_timestep_latent_bounds():
    g = torch.Generator().manual_seed(4)
    x, w = torch.randn(9, 320, generator=g), (torch.randn(7, 320, generator=g) * 320 ** -0.5).half()
    b, a = torch.randn(7, generator=g), torch.randn(7, generator=g)
    for act_in, act_out in ((False, False), (True, True)):
        ref, tol = OR.linear_small(x, w, b, a, act_in, act_out)
        xi = x * torch.sigmoid(x) if act_in else x
        y = xi @ w.float().t() + (b + a)
        emu = y * torch.sigmoid(y) if act_out else y
        assert OR.worst(emu, ref, tol) <= 1.0
        assert OR.rejects(OR.linear_small(x, w, b, a, act_in, act_out, drop_last_k=True)[0], ref, tol)
    t = torch.tensor([1.0, 501.0, 999.0])
    ref, tol = OR.timestep_embedding(t, 320, True, 1.0)
    half = 160
    freq = torch.exp(-torch.log(torch.tensor(10000.0)) * torch.arange(half).float() / (half - 1.0))
    ang = t[:, None] * freq
    assert OR.worst(torch.cat([torch.cos(ang), torch.sin(ang)], -1), ref, tol) <= 1.0
    assert OR.rejects(OR.timestep_embedding(t, 320, True, 1.0, perturb=True)[0], ref, tol)
    z, wq, bq = torch.randn(1, 4, 5, 6, generator=g), torch.randn(4, 4, generator=g), torch.randn(4, generator=g)
    ref, tol = OR.latent_prep(z, wq, bq, 0.5, 8, BF16)
    emu = torch.zeros(1, 5, 6, 8)
    emu[..., :4] = (z * 0.5).permute(0, 2, 3, 1) @ wq.t() + bq
    assert OR.worst(emu.to(BF16), ref, tol) <= 1.0
    assert OR.rejects(OR.latent_prep(z, wq, bq, 0.5, 8, BF16, drop_last=True)[0], ref, tol)


@pytest.mark.parametrize("sk,causal", [(77, False), (300, False), (300, True)])
def test_attention_bound(sk, causal):
    """fp32 scores, probabilities rounded to fp16 before P V, fp16 output: accepted; the last key or the first K/V tile
    left out: rejected.  Views with a row stride, as the models pass them."""
    g = torch.Generator().manual_seed(5)
    batch, heads, d, sq = 2, 2, 40, 130 if causal else 33
    sk = sq if causal else sk
    qkv = torch.randn(batch * max(sq, sk), 3 * heads * d + 8, generator=g).half()
    q, k, v = qkv[:batch * sq, :heads * d], qkv[:batch * sk, heads * d:2 * heads * d], qkv[:batch * sk, 2 * heads * d:-8]
    out = torch.empty(batch * sq, heads * d, dtype=F16)
    for b in range(batch):
        for h in range(heads):
            c = slice(h * d, (h + 1) * d)
            s = (q[b * sq:(b + 1) * sq, c].float() @ k[b * sk:(b + 1) * sk, c].float().t()) * d ** -0.5
            if causal:
                s = s.masked_fill(torch.ones(sq, sk, dtype=torch.bool).triu(1), float("-inf"))
            p = torch.exp(s - s.max(-1, keepdim=True).values)
            o = p.half().float() @ v[b * sk:(b + 1) * sk, c].float() / p.sum(-1, keepdim=True)
            out[b * sq:(b + 1) * sq, c] = o.half()
    w, wl, wt = OR.attention_check(q, k, v, out, batch, heads, sq, sk, d, d ** -0.5, causal=causal, kv_tile=128,
                                   max_elems=4096)
    assert w <= 1.0 and wl > 1.0 and (wt is None or wt > 1.0), (w, wl, wt)


def test_image_postprocess_reference():
    x = torch.tensor([-3.0, -1.0, -0.999, 0.0, 0.001, 0.5, 1.0, 7.0]).reshape(1, 1, 1, 8)
    img = OR.image_postprocess(x, 8)
    assert img.min() == 0.0 and img.max() == 1.0
    assert OR.to_u8(img).tolist() == [[[[0, 0, 0, 128, 128, 191, 255, 255]]]]


@pytest.mark.parametrize("fn", ["nhwc_to_nchw_f32", "image_postprocess", "ctx_to_tokens"])
@pytest.mark.parametrize("dt", [torch.bfloat16, torch.float64, torch.int16])
def test_fp16_fp32_only_wrappers_reject_other_types(fn, dt):
    """These kernels take one fp16 / fp32 flag: any other type would be read as fp16 bits, so the wrapper refuses it
    (checked before the library is touched, so no device is needed)."""
    from b200sd import lib

    x = torch.zeros(1, 8, 1, 8, dtype=dt)
    with pytest.raises(lib.B200SDError, match=str(dt).replace("torch.", "")):
        getattr(lib, fn)(x)
