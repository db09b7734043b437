"""GPU tests of every attention, normalisation and elementwise launch of the shipped models, and of the shapes the models
do not reach, against an fp64 reference of that one launch (op_refs.py; test_op_refs.py rehearses every bound on the
CPU).  The GEMM / convolution kernels have test_gemm_plans_gpu.py.

Replay.  lib.attention, group_norm, group_norm_apply, layer_norm, softmax_rows, linear_small, timestep_embedding,
embed_tokens, ctx_to_tokens, add, upsample2x, nchw_to_nhwc, nhwc_to_nchw_f32 and latent_prep are wrapped: the inputs
are cloned before the launch (the `out=` buffers may alias them, as in L.add(acc, o, out=acc); a strided view is cloned
with its strides, so the attention reference reads the fused QKV / kv_all views the kernel read), the call runs as
usual, runs once more on the clones into a fresh output and must be bit-identical (stream-K merges, cluster exchanges,
GroupNorm tickets), then is compared with the reference.  A GroupNorm launch is the cluster kernel when it counted one
launch and the two-kernel fallback when it counted two.

Exact ops must be bit-identical to their reference: upsample2x, the layout conversions and ctx_to_tokens are copies or
one correctly rounded conversion; add rounds the fp32 sum of two fp16 values (exact up to one rounding to 24 bits, and
24 >= 2 * 11 + 2 makes the second rounding innocuous) and embed_tokens uses __hadd2: both equal (a + b) in fp64 rounded
once to fp16.

Bounds.  Per element |got - ref| <= r_out |ref| + tau * B with B the same computation on magnitudes, r_out = 2^-10
(fp16) / 2^-7 (bf16), twice the unit roundoff, as in the GEMM tests, and an activation's Lipschitz bound 1.13:
  * GroupNorm / LayerNorm: the statistics are fp32 sums with relative error E (E = 2^-18 for the kernels' own sums:
    fixed-order sums of up to a few hundred terms per chain, random-signed 2^-24 per addition; E = 2^-14 for the
    producers' per-channel sums group_norm_apply folds, the bound test_gemm_plans_gpu.py asserts for them).  One-pass
    E[x^2] - mean^2 (GroupNorm) is off by E (mu^2 + sigma^2), a relative variance error E (1 + (mu / sigma)^2) and half
    that on rstd; the mean is off by E (1 + |mu| / sigma) sigma.  B = |gamma| (|x_hat| (1 + rho^2) / 2 + 1 + rho),
    rho = |mu| / sigma per group, tau = E, times 1.13 with SiLU (whose __expf / __fdividef add 2^-19 relative).
    LayerNorm is two-pass: the mean error enters the variance only squared, E + E^2 (1 + rho)^2.
  * softmax_rows: relative r_out + 2^-18 + 2^-24 (2 |z| + 2 max |z| + 4), z the scaled scores in the exp2 domain.
  * attention: r_out |ref| + 8 R (2^-11 + (d + 2) 2^-24 S) + 2^-20 P |V|, with R = sqrt(sum_j P_j^2 V_j^2): the fp16
    probabilities and the score errors are random-signed over the keys (see op_refs.attention_check).
  * linear_small: 2^-20 (|x| . |w|^T + |bias| + |add|), SiLU as above; timestep embedding: 2^-18 |t freq| + 2^-21.
Sensitivity.  Every bound must reject a perturbed reference: GroupNorm statistics over group boundaries moved by one
8-channel vector (and, in the synthetic cases, statistics missing the last CTA's or chunk's pixels, visible through a
spatial ramp in the input); LayerNorm statistics over rows moved by 8 channels; softmax without its last column;
attention without its last key and without its first K/V tile; linear_small without its last 8 input features; the
embedding with its frequency table shifted by one; latent_prep without its last input channel.

Run with -s for one line per distinct (op, shape, dtype, path) with its launch count and worst err / tol."""
import os
import sys
import time

import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import model_cases as MC  # noqa: E402
import op_refs as OR  # noqa: E402

pytestmark = pytest.mark.gpu

F16, BF16, F32 = torch.float16, torch.bfloat16, torch.float32
KV_TILE = {40: 128, 64: 128, 80: 128, 160: 64}  # keys per K/V tile (attention.cu AttnKeys)


def _clone(t):
    """A copy of t with t's strides (a strided view stays a strided view); non-tensors pass through."""
    if not isinstance(t, torch.Tensor):
        return t
    if t.is_contiguous():
        return t.clone()
    span = 1 + sum((s - 1) * st for s, st in zip(t.shape, t.stride()))
    return t.as_strided((span,), (1,)).clone().as_strided(t.shape, t.stride())


def _nhwc(x, x1=None):
    xx = x if x1 is None else torch.cat([x, x1], -1)
    return xx.double().reshape(xx.shape[0], -1, xx.shape[-1])


def _dt(t):
    return {F16: "fp16", BF16: "bf16", F32: "fp32"}[t]


class _Replay:
    OPS = ("attention", "group_norm", "group_norm_apply", "layer_norm", "softmax_rows", "linear_small",
           "timestep_embedding", "embed_tokens", "ctx_to_tokens", "add", "upsample2x", "nchw_to_nhwc",
           "nhwc_to_nchw_f32", "latent_prep")

    def __init__(self, lib, model):
        self.lib, self.model = lib, model
        self.rows = {}  # (op, shape, dtype, path) -> (launches, worst err / tol)

    def install(self, monkeypatch):
        for op in self.OPS:
            monkeypatch.setattr(self.lib, op, self._wrap(op, getattr(self.lib, op), getattr(self, "_" + op)))

    def _wrap(self, op, f0, check):
        def call(*a, **kw):
            ca = [_clone(t) for t in a]
            ckw = {k: _clone(v) for k, v in kw.items()}
            n0 = self.lib.launch_count()
            y = f0(*a, **kw)
            launches = self.lib.launch_count() - n0
            rkw = dict(ckw)
            if kw.get("out") is not None:
                rkw["out"] = torch.empty_like(kw["out"])
            y2 = f0(*ca, **rkw)
            torch.cuda.synchronize()
            for u, u2 in zip(y if isinstance(y, tuple) else (y,), y2 if isinstance(y2, tuple) else (y2,)):
                assert torch.equal(u, u2), f"{self.model} {op}: a second identical launch differs"
            key, w = check(launches, y, *ca, **ckw)
            n, w0 = self.rows.get(key, (0, 0.0))
            self.rows[key] = (n + 1, max(w0, w))
            assert w <= 1.0, f"{self.model} {key}: worst err/tol {w:.3g}"
            return y
        return call

    # ---- the checks: (table key, worst err / tol); each asserts its sensitivity probe ----
    def _attention(self, launches, y, q, k, v, batch, heads, sq, sk, d=64, mask=None, impl=0, out=None, scale=None,
                   causal=False):
        sc = float(d) ** -0.5 if scale is None else float(scale)
        w, wl, wt = OR.attention_check(q, k, v, y, batch, heads, sq, sk, d, sc, mask=mask, causal=causal,
                                       kv_tile=KV_TILE[d])
        what = f"{self.model} attention b={batch} h={heads} sq={sq} sk={sk} d={d}"
        assert wl > 1.0, f"{what}: the bound cannot see the last key missing ({wl:.3g})"
        assert wt is None or wt > 1.0, f"{what}: the bound cannot see the first K/V tile missing ({wt:.3g})"
        path = "causal" if causal else ("mask" if mask is not None else "-")
        return ("attention", (batch, heads, sq, sk, d), "fp16", path), w

    def _gn_check(self, op, launches, y, x, x1, gamma, beta, groups, eps, silu, e_sum):
        xd = _nhwc(x, x1)
        dt = x.dtype
        ref, tol = OR.group_norm(xd, gamma, beta, groups, eps, silu, dt, e_sum=e_sum)
        w = OR.worst(y.reshape(xd.shape), ref, tol)
        alt = OR.group_norm(xd, gamma, beta, groups, eps, silu, dt, e_sum=e_sum, stats=OR.gn_stats(xd, groups, shift=8))[0]
        assert OR.rejects(alt, ref, tol), f"{self.model} {op} {tuple(xd.shape)}: bound blind to shifted groups"
        path = "producer" if op == "group_norm_apply" else {1: "cluster", 2: "fallback"}[launches]
        c0 = x.shape[-1]
        shape = (x.shape[0], x.shape[1], x.shape[2], c0 if x1 is None else f"{c0}+{x1.shape[-1]}", groups)
        return (op, shape, _dt(dt), path + (" silu" if silu else "")), w

    def _group_norm(self, launches, y, x, gamma, beta, groups, eps, silu=False, x1=None, out=None):
        return self._gn_check("group_norm", launches, y, x, x1, gamma, beta, groups, eps, silu, OR.E_SUM)

    def _group_norm_apply(self, launches, y, x, chan0, gamma, beta, groups, eps, silu=False, x1=None, chan1=None,
                          out=None):
        return self._gn_check("group_norm_apply", launches, y, x, x1, gamma, beta, groups, eps, silu, OR.E_PRODUCER)

    def _layer_norm(self, launches, y, x, gamma, beta, eps=1e-5, out=None):
        ref, tol = OR.layer_norm(x.double(), gamma, beta, eps)
        if x.shape[0] > 1:
            assert OR.rejects(OR.layer_norm(x.double(), gamma, beta, eps, shift=8)[0], ref, tol), "layer_norm probe"
        return ("layer_norm", tuple(x.shape), "fp16", "-"), OR.worst(y, ref, tol)

    def _softmax_rows(self, launches, y, scores, scale, out=None, out_dtype=F16):
        ref, tol = OR.softmax_rows(scores, scale, y.dtype)
        if float(ref[:, -1].max()) > 2.0 ** -20:  # one-hot rows leave nothing in the last column to miss
            assert OR.rejects(OR.softmax_rows(scores, scale, y.dtype, drop_last=True)[0], ref, tol), "softmax probe"
        return ("softmax_rows", tuple(scores.shape), _dt(y.dtype), "-"), OR.worst(y, ref, tol)

    def _linear_small(self, launches, y, x, wgt, bias=None, add=None, act_in=False, act_out=False):
        ref, tol = OR.linear_small(x, wgt, bias, add, act_in, act_out)
        alt = OR.linear_small(x, wgt, bias, add, act_in, act_out, drop_last_k=True)[0]
        assert OR.rejects(alt, ref, tol), "linear_small probe"
        path = "".join(f for f, on in (("b", bias is not None), ("+", add is not None), ("i", act_in), ("o", act_out))
                       if on) or "-"
        return ("linear_small", (x.shape[0], wgt.shape[1], wgt.shape[0]), "fp32", path), OR.worst(y, ref, tol)

    def _timestep_embedding(self, launches, y, t, dim, flip_sin_to_cos=True, freq_shift=0.0):
        ref, tol = OR.timestep_embedding(t, dim, flip_sin_to_cos, freq_shift)
        assert OR.rejects(OR.timestep_embedding(t, dim, flip_sin_to_cos, freq_shift, perturb=True)[0], ref, tol)
        return ("timestep_embedding", (t.shape[0], dim), "fp32", "-"), OR.worst(y, ref, tol)

    def _latent_prep(self, launches, y, z, w, b, inv_scale, c_pad=8, out_dtype=F16):
        ref, tol = OR.latent_prep(z, w, b, inv_scale, c_pad, y.dtype)
        if z.shape[1] > 1:
            assert OR.rejects(OR.latent_prep(z, w, b, inv_scale, c_pad, y.dtype, drop_last=True)[0], ref, tol)
        return ("latent_prep", tuple(z.shape), _dt(y.dtype), "-"), OR.worst(y, ref, tol)

    # ---- exact ops: bit-identical ----
    def _exact(self, op, y, ref, shape, dt):
        assert y.dtype == ref.dtype and torch.equal(y, ref), f"{self.model} {op} {shape}: not bit-identical"
        return (op, shape, dt, "exact"), 0.0

    def _embed_tokens(self, launches, y, ids, tok, pos, out=None):
        b, s = ids.shape
        idx = torch.round(ids).clamp(0, tok.shape[0] - 1).long()
        ref = (tok[idx].double() + pos[:s].double()[None]).reshape(b * s, -1).half()
        return self._exact("embed_tokens", y, ref, (b, s, tok.shape[1]), "fp16")

    def _ctx_to_tokens(self, launches, y, ctx, out=None):
        b, d, _, s = ctx.shape
        ref = ctx[:, :, 0, :].permute(0, 2, 1).reshape(b * s, d).half()
        return self._exact("ctx_to_tokens", y, ref, tuple(ctx.shape), _dt(ctx.dtype))

    def _add(self, launches, y, a, b, out=None):
        return self._exact("add", y, (a.double() + b.double()).half(), tuple(a.shape), "fp16")

    def _upsample2x(self, launches, y, x, out=None):
        ref = x.repeat_interleave(2, 1).repeat_interleave(2, 2)
        return self._exact("upsample2x", y, ref, tuple(x.shape), _dt(x.dtype))

    def _nchw_to_nhwc(self, launches, y, x, c_pad=None, out=None, out_dtype=F16):
        n, c, h, w = x.shape
        ref = torch.zeros(n, h, w, y.shape[-1], dtype=y.dtype, device=x.device)
        ref[..., :c] = x.permute(0, 2, 3, 1).to(y.dtype)
        return self._exact("nchw_to_nhwc", y, ref, (tuple(x.shape), y.shape[-1]), f"{_dt(x.dtype)}->{_dt(y.dtype)}")

    def _nhwc_to_nchw_f32(self, launches, y, x, c=None, out=None):
        c = x.shape[-1] if c is None else c
        ref = x[..., :c].permute(0, 3, 1, 2).float().contiguous()
        return self._exact("nhwc_to_nchw_f32", y, ref, (tuple(x.shape), c), _dt(x.dtype))

    def report(self):
        lines = [f"{self.model}: {sum(v[0] for v in self.rows.values())} launches, {len(self.rows)} distinct"]
        for (op, shape, dt, path), (n, w) in sorted(self.rows.items(), key=str):
            lines.append(f"  {op:18s} {str(shape):34s} {dt:10s} {path:16s} x{n:<4d} worst err/tol {w:.3f}")
        return "\n".join(lines)


MODELS = MC.SHIPPED + ["sd21_b2_fused2", "sd15_512x768_b2_fused2"]


def _gn_channels(rows):
    """Total channels of every GroupNorm row of a report (shape key (n, h, w, C0 or "C0+C1", groups))."""
    return {sum(int(c) for c in str(key[1][3]).split("+")) for key in rows if key[0].startswith("group_norm")}


@pytest.mark.parametrize("name", MODELS)
def test_model_op_launches_match_fp64_reference(cuda_lib, monkeypatch, name):
    """One eager forward of each model of model_cases.SHIPPED (*_fused2: SD-2.1 and SD-1.5 at 512x768 under
    B200SD_FUSED=2, where group_norm_apply normalises from the producers' channel sums), every wrapped launch checked.
    Prints the table and the wall time of the build, forward and checks (run with -s)."""
    lib = cuda_lib
    for k in ("B200SD_CLUSTER_SPLITK", "B200SD_STAGED", "B200SD_FUSED", "B200SD_HALO_TMA"):
        monkeypatch.delenv(k, raising=False)
    if name.endswith("_fused2"):
        monkeypatch.setenv("B200SD_FUSED", "2")
    t0 = time.perf_counter()
    m = MC.build(name[: -len("_fused2")] if name.endswith("_fused2") else name)
    rep = _Replay(lib, name)
    rep.install(monkeypatch)
    m(**MC.model_inputs(m, seed=9))
    torch.cuda.synchronize()
    print(f"\n{rep.report()}\n  wall time {time.perf_counter() - t0:.1f} s")
    ops = {key[0] for key in rep.rows}
    assert rep.rows, f"{name}: no launch was seen"
    if name.startswith(("sd", "controlnet")):
        gn = "group_norm_apply" if name.endswith("_fused2") else "group_norm"
        assert {"attention", gn, "linear_small", "timestep_embedding"} <= ops, sorted(ops)
    if name.startswith("vae_decoder"):
        assert {"group_norm", "softmax_rows", "latent_prep", "upsample2x"} <= ops, sorted(ops)
    if name.startswith("vae_encoder"):
        assert {"group_norm", "softmax_rows"} <= ops, sorted(ops)
    if name.startswith(("openclip", "clip")):
        assert {"attention", "layer_norm", "embed_tokens"} <= ops, sorted(ops)
    # the shapes each new case exists for
    if name.startswith("sdxl_refiner"):  # groups of 12, 36 and 96 channels: none a whole number of 8-channel vectors
        assert {384, 1152, 3072} <= _gn_channels(rep.rows), sorted(_gn_channels(rep.rows))
        assert {key[1][4] for key in rep.rows if key[0] == "attention"} == {64}
    if name.startswith(("controlnet_sd15", "sd15")):
        assert {key[1][4] for key in rep.rows if key[0] == "attention"} == {40, 80, 160}
    if name.endswith("_768") and name.startswith("vae_decoder"):
        assert any(key[0] == "softmax_rows" and key[1][1] == 96 * 96 for key in rep.rows)
        assert any(key[0] == "group_norm" and key[1][1:3] == (768, 768) for key in rep.rows)
    # the non-square and odd maps: the deepest map and the attention token counts each size exists for
    gn_maps = {tuple(key[1][1:3]) for key in rep.rows if key[0].startswith("group_norm")}
    tokens = {key[1][2] for key in rep.rows if key[0] == "attention"}
    want = NON_SQUARE_SHAPES.get(name[: -len("_fused2")] if name.endswith("_fused2") else name)
    if want is not None:
        assert want["maps"] <= gn_maps, (sorted(want["maps"]), sorted(gn_maps))
        assert want.get("tokens", set()) <= tokens, (sorted(want.get("tokens", set())), sorted(tokens))
        if "softmax" in want:
            assert any(key[0] == "softmax_rows" and key[1][1] == want["softmax"] for key in rep.rows), sorted(rep.rows)


# (h, w) maps some GroupNorm of the model must run on, attention query counts it must reach, softmax_rows columns
NON_SQUARE_SHAPES = {
    "sd15_512x768_b2": dict(maps={(64, 96), (8, 12)}, tokens={6144, 1536, 384, 96}),
    "sd15_768x512_b2": dict(maps={(96, 64), (12, 8)}, tokens={6144, 1536, 384, 96}),
    "sd21_576x576_b2": dict(maps={(72, 72), (18, 18), (9, 9)}, tokens={5184, 1296, 324, 81}),
    "sdxl_768x1344_b2": dict(maps={(96, 168), (24, 42)}, tokens={4032, 1008}),
    "sdxl_1216x832_b2": dict(maps={(152, 104), (38, 26)}, tokens={3952, 988}),
    "sdxl_refiner_768x1344_b2": dict(maps={(96, 168), (12, 21)}, tokens={4032, 1008, 252}),
    "controlnet_sd15_512x768": dict(maps={(64, 96), (8, 12)}, tokens={6144, 96}),
    "vae_decoder_512x768": dict(maps={(64, 96), (512, 768)}, softmax=64 * 96),
    "vae_decoder_bf16_768x1344": dict(maps={(96, 168), (768, 1344)}, softmax=96 * 168),
    "vae_encoder_768x512": dict(maps={(768, 512), (96, 64)}, softmax=96 * 64),
    "vae_encoder_bf16_1216x832": dict(maps={(1216, 832), (152, 104)}, softmax=152 * 104),
}


# ---------------------------------------------------------------------------------------------------------------------
# Synthetic edge cases the models do not reach.
# ---------------------------------------------------------------------------------------------------------------------
def _gn_input(g, n, hw, c, groups, rho, dt, dev="cuda"):
    """randn + a per-group offset of +-rho (so |mu| / sigma ~ rho), alternating in sign so that every group boundary
    separates offsets 2 rho apart (a boundary moved by 8 channels shows at any group width) + a spatial ramp (pixel
    range errors show)."""
    sign = 1.0 - 2.0 * (torch.arange(groups, device=dev) % 2)
    off = (rho * sign).repeat_interleave(c // groups)
    ramp = torch.linspace(-1.0, 1.0, hw, device=dev)[None, :, None]
    return (torch.randn(n, hw, c, generator=g, device=dev) + off + ramp).to(dt)


def _gn_run(lib, x, c0, h, w, groups, silu, dt, rho, drop_px, expect_launches, gamma=None, beta=None):
    """One group_norm launch of x [n, hw, C] split into sources c0 | C - c0; checks launches, repeatability, the bound
    and both probes; returns worst err / tol."""
    n, hw, c = x.shape
    g = torch.Generator(device="cuda").manual_seed(c + hw)
    gamma = 1 + 0.2 * torch.randn(c, generator=g, device="cuda") if gamma is None else gamma
    beta = 0.1 * torch.randn(c, generator=g, device="cuda") if beta is None else beta
    x4 = x.reshape(n, h, w, c)
    xa, xb = x4[..., :c0].contiguous(), (x4[..., c0:].contiguous() if c0 < c else None)
    n0 = lib.launch_count()
    y = lib.group_norm(xa, gamma, beta, groups, 1e-5, silu=silu, x1=xb)
    assert lib.launch_count() - n0 == expect_launches, (n, hw, c, groups)
    y2 = lib.group_norm(xa, gamma, beta, groups, 1e-5, silu=silu, x1=xb)
    torch.cuda.synchronize()
    assert torch.equal(y, y2)
    xd = x.double()
    ref, tol = OR.group_norm(xd, gamma, beta, groups, 1e-5, silu, dt)
    w_ = OR.worst(y.reshape(n, hw, c), ref, tol)
    assert w_ <= 1.0, f"GroupNorm n={n} hw={hw} C={c0}+{c - c0} groups={groups} rho={rho} {dt}: err/tol {w_:.3g}"
    probes = [("last pixels missing", OR.gn_stats(xd, groups, px=slice(0, hw - drop_px)))] if drop_px else []
    if groups > 1:
        probes.append(("groups shifted by 8 channels", OR.gn_stats(xd, groups, shift=8)))
    for what, st in probes:
        assert OR.rejects(OR.group_norm(xd, gamma, beta, groups, 1e-5, silu, dt, stats=st)[0], ref, tol), \
            f"GroupNorm n={n} hw={hw} C={c} groups={groups}: the bound cannot see {what}"
    return w_


def _fallback_last_chunk(hw):
    """Pixels of the last non-empty statistics chunk of the fallback (norm.cu gn_chunks: min(128, hw / 16) chunks of
    ceil(hw / chunks) pixels)."""
    chunks = max(1, min(128, hw // 16))
    ppc = -(-hw // chunks)
    return hw - (hw - 1) // ppc * ppc


@pytest.mark.parametrize("dt", [F16, BF16])
@pytest.mark.parametrize("groups,c,hw", [(1, 520, 1039), (1, 520, 2049), (1, 520, 2048), (2, 1040, 1039),
                                         (2, 1040, 2049), (2, 1040, 2048), (2, 3072, 1039), (2, 3072, 2049),
                                         (32, 3072, 8193)])
def test_group_norm_fallback_empty_chunks(cuda_lib, dt, groups, c, hw):
    """A chunk of > 512 channels is refused by the cluster planner, so these run the two-kernel fallback.  hw = 1039:
    64 chunks of 17 pixels, the last two empty; hw = 2049: 128 chunks of 17, the last seven empty; hw = 2048: 128 full
    chunks (the control).  C = 3072 is the SDXL refiner's widest concatenation (1536 + 1536), 384 vectors per pixel:
    the most the fallback takes.  At 32 groups of 96 channels and hw = 8193 the cluster path is refused for its slab
    (1025 rows x 192 B > 200 KB at cluster size 8, 2 at 5 images) and the fallback runs 128 chunks of 65 pixels, the
    last one empty.  2 images, then 5: the ticket counters reset themselves between launches."""
    lib = cuda_lib
    g = torch.Generator(device="cuda").manual_seed(hw + groups)
    for n in (2, 5):
        x = _gn_input(g, n, hw, c, groups, 3.0, dt)
        _gn_run(lib, x, c // 2 // 8 * 8, hw, 1, groups, True, dt, 3.0, _fallback_last_chunk(hw), 2)


# (C0, C1, h, w, images) -> cluster size and rows in flight as norm.cu plans them on a 132-SM H100 (chunk = lcm(C/32, 8)
# widened to >= 32 channels; cs = 8 halved while hw / cs < 32 or clusters * cs > 4 * SMs; deep (8 rows in flight) when
# a thread has >= 3 rows):
CLUSTER_CASES = [
    (320, 0, 64, 64, 2),       # cs 8, deep; 512 rows per CTA
    (640, 320, 27, 37, 2),     # cs 8, deep; ragged (125 x 7 + 124 rows); group 21 straddles the c0 / c1 boundary
    (1280, 1280, 24, 24, 2),   # cs 8, deep; C = 2560 (SDXL up blocks)
    (1280, 0, 16, 16, 3),      # cs 4, 2 rows in flight
    (1280, 0, 12, 12, 2),      # cs 4, 2 rows in flight; the 768-v lowest level
    (1280, 0, 15, 17, 6),      # cs 2, deep; ragged (128 + 127 rows)
    (1280, 0, 16, 16, 16),     # cs 1, deep; batch 16
    (320, 0, 6, 6, 2),         # cs 1, 2 rows in flight
    # the SDXL refiner's geometries: groups of 12, 36, 96 and 72 channels, none a whole number of 8-channel vectors
    (384, 0, 128, 128, 2),     # chunk 48 (lcm(12, 8) = 24, doubled to >= 32), 6 vectors: 2048 rows per CTA at cs 8 make
                               # a 213 KB slab > 200 KB, so the planner refuses it: the fallback (cs 0, two launches)
    (768, 384, 64, 64, 2),     # cs 8, deep; chunk 72 = lcm(36, 8), 9 vectors, 28 rows x 9 = 252 of 256 threads
    (1536, 1536, 32, 32, 2),   # cs 8, deep; C = 3072, chunk 96, 12 vectors, 21 rows x 12 = 252 threads
    (1536, 768, 16, 16, 2),    # cs 8, 2 rows in flight; C = 2304, chunk 72, 32 rows per CTA
    (1536, 1536, 12, 12, 2),   # cs 4, 2 rows in flight; the refiner's lowest level at 768^2 (hw / 8 = 18 < 32)
    (1536, 1536, 32, 32, 16),  # 512 clusters: cs 1, whose 1024-row slab (209 KB) is refused: the fallback at C = 3072,
                               # 384 vectors, one row: 48 KB of dynamic shared memory beside the kernel's static ticket
                               # (the refiner at 1024^2, 8 images per call)
]
CLUSTER_SIZE = [8, 8, 8, 4, 4, 2, 1, 1, 0, 8, 8, 8, 4, 0]


@pytest.mark.parametrize("dt", [F16, BF16])
@pytest.mark.parametrize("case", range(len(CLUSTER_CASES)))
def test_group_norm_cluster_shapes(cuda_lib, dt, case):
    """Cluster size 0: the planner refuses the cluster kernel and the two-kernel fallback runs; its probe drops the last
    statistics chunk's pixels."""
    lib = cuda_lib
    c0, c1, h, w, n = CLUSTER_CASES[case]
    cs, hw, c = CLUSTER_SIZE[case], h * w, c0 + c1
    g = torch.Generator(device="cuda").manual_seed(case)
    x = _gn_input(g, n, hw, c, 32, 3.0, dt)
    if cs == 0:
        _gn_run(lib, x, c0, h, w, 32, case % 2 == 0, dt, 3.0, _fallback_last_chunk(hw), 2)
        return
    drop = hw - (cs - 1) * (-(-hw // cs)) if cs > 1 else 0  # the last CTA's pixels
    _gn_run(lib, x, c0, h, w, 32, case % 2 == 0, dt, 3.0, drop, 1)


@pytest.mark.parametrize("dt", [F16, BF16])
@pytest.mark.parametrize("rho", [0.0, 10.0, 30.0])
@pytest.mark.parametrize("path", ["cluster", "fallback"])
def test_group_norm_mean_offset(cuda_lib, dt, rho, path):
    """|mu| / sigma up to 30 against the one-pass bound, on both paths."""
    lib = cuda_lib
    g = torch.Generator(device="cuda").manual_seed(int(rho) + 7)
    if path == "cluster":
        x = _gn_input(g, 2, 4096, 320, 32, rho, dt)
        _gn_run(lib, x, 320, 64, 64, 32, False, dt, rho, 512, 1)
    else:
        x = _gn_input(g, 2, 4096, 1040, 2, rho, dt)
        _gn_run(lib, x, 1040, 64, 64, 2, False, dt, rho, _fallback_last_chunk(4096), 2)


@pytest.mark.parametrize("rho", [0.0, 10.0])
def test_group_norm_apply_producer_sums(cuda_lib, rho):
    """group_norm_apply folds the producers' fp32 channel sums: its bound is the one-pass bound at E = 2^-14 (the
    producers' sums' own bound), so it is tested at |mu| / sigma <= 10 with sums of that quality (fp64 sums rounded
    to fp32 are far better), over a c0 / c1 boundary inside a group."""
    lib = cuda_lib
    g = torch.Generator(device="cuda").manual_seed(int(rho) + 11)
    n, h, w, c0, c1, groups = 2, 32, 32, 640, 320, 32
    x = _gn_input(g, n, h * w, c0 + c1, groups, rho, F16)
    gamma, beta = 1 + 0.2 * torch.randn(c0 + c1, generator=g, device="cuda"), 0.1 * torch.randn(c0 + c1, generator=g,
                                                                                                   device="cuda")
    x4 = x.reshape(n, h, w, -1)
    xa, xb = x4[..., :c0].contiguous(), x4[..., c0:].contiguous()

    def sums(t):
        td = t.double().reshape(n, -1, t.shape[-1])
        return torch.stack([td.sum(1), (td * td).sum(1)], -1).float().contiguous()

    y = lib.group_norm_apply(xa, sums(xa), gamma, beta, groups, 1e-5, silu=True, x1=xb, chan1=sums(xb))
    xd = x.double()
    ref, tol = OR.group_norm(xd, gamma, beta, groups, 1e-5, True, F16, e_sum=OR.E_PRODUCER)
    assert OR.worst(y.reshape(xd.shape), ref, tol) <= 1.0
    alt = OR.group_norm(xd, gamma, beta, groups, 1e-5, True, F16, e_sum=OR.E_PRODUCER,
                        stats=OR.gn_stats(xd, groups, shift=8))[0]
    assert OR.rejects(alt, ref, tol)


@pytest.mark.parametrize("c", [8, 256, 512, 520, 1280, 1288, 2048])
def test_layer_norm_shapes(cuda_lib, c):
    """Each kVecsPerLane instantiation (2: C <= 512, 5: <= 1280, 8: <= 2048) and its boundaries; a mean offset of 100."""
    lib = cuda_lib
    g = torch.Generator(device="cuda").manual_seed(c)
    gamma, beta = 1 + 0.2 * torch.randn(c, generator=g, device="cuda"), 0.1 * torch.randn(c, generator=g, device="cuda")
    for rows in (1, 7, 9, 154, 8193):
        x = (100 + torch.randn(rows, c, generator=g, device="cuda")).half()
        y = lib.layer_norm(x, gamma, beta)
        y2 = lib.layer_norm(x, gamma, beta)
        assert torch.equal(y, y2)
        ref, tol = OR.layer_norm(x.double(), gamma, beta, 1e-5)
        assert OR.worst(y, ref, tol) <= 1.0, (rows, c)
        if rows > 1:
            assert OR.rejects(OR.layer_norm(x.double(), gamma, beta, 1e-5, shift=8)[0], ref, tol), (rows, c)


def test_linear_small_shapes(cuda_lib):
    """m in {1, 2, 3, 8, 9, 17, 32} (row chunks of 8 through <8>, a last chunk of 1 or 2 rows through <2>), k in
    {8, 320, 1288, 2816}, n in {1, 7, 1280}, bias / add / act_in / act_out cycling through all 16 combinations."""
    lib = cuda_lib
    g = torch.Generator(device="cuda").manual_seed(3)
    i = 0
    seen = set()
    for m in (1, 2, 3, 8, 9, 17, 32):
        for k in (8, 320, 1288, 2816):
            for n in (1, 7, 1280):
                fl = [(i >> b) & 1 for b in range(4)]
                i += 1
                x = torch.randn(m, k, generator=g, device="cuda")
                w = (torch.randn(n, k, generator=g, device="cuda") * k ** -0.5).half()
                bias = torch.randn(n, generator=g, device="cuda") if fl[0] else None
                add = torch.randn(n, generator=g, device="cuda") if fl[1] else None
                y = lib.linear_small(x, w, bias, add, act_in=bool(fl[2]), act_out=bool(fl[3]))
                assert torch.equal(y, lib.linear_small(x, w, bias, add, act_in=bool(fl[2]), act_out=bool(fl[3])))
                ref, tol = OR.linear_small(x, w, bias, add, fl[2], fl[3])
                assert OR.worst(y, ref, tol) <= 1.0, (m, k, n, fl)
                alt = OR.linear_small(x, w, bias, add, fl[2], fl[3], drop_last_k=True)[0]
                assert OR.rejects(alt, ref, tol), (m, k, n, fl)
                seen.add(tuple(fl))
    assert len(seen) == 16


@pytest.mark.parametrize("dt", [F16, BF16])
@pytest.mark.parametrize("cols", [1, 7, 255, 256, 257, 4096, 16384])
def test_softmax_rows_shapes(cuda_lib, dt, cols):
    """Random rows, a row with one dominant entry, and scales from 1e-6 to 300."""
    lib = cuda_lib
    g = torch.Generator(device="cuda").manual_seed(cols)
    s = torch.randn(5, cols, generator=g, device="cuda")
    s[1, cols // 2] = 40.0
    for scale in (1e-6, 0.044, 1.0, 300.0):
        y = lib.softmax_rows(s, scale, out_dtype=dt)
        assert torch.equal(y, lib.softmax_rows(s, scale, out_dtype=dt))
        ref, tol = OR.softmax_rows(s, scale, dt)
        assert OR.worst(y, ref, tol) <= 1.0, (cols, scale)
        if cols > 1 and scale < 1:  # at scale 300 the rows are one-hot: the last column holds nothing to miss
            assert OR.rejects(OR.softmax_rows(s, scale, dt, drop_last=True)[0], ref, tol), (cols, scale)


@pytest.mark.parametrize("d", [40, 64, 80, 160])
def test_attention_edges(cuda_lib, d):
    """sk in {1, 2, KV - 1, KV + 1} x sq in {1, 127, 129} on strided views of one fused buffer (the models' QKV
    layout), one case at a non-default scale; then a mask that leaves one visible key per image."""
    lib = cuda_lib
    kv = KV_TILE[d]
    batch, heads = 2, 2
    g = torch.Generator(device="cuda").manual_seed(d)
    for sk in (1, 2, kv - 1, kv + 1):
        for sq in (1, 127, 129):
            rows = batch * max(sq, sk)
            buf = torch.randn(rows, 3 * heads * d + 8, generator=g, device="cuda").half()
            q, k, v = (buf[:batch * sq, :heads * d], buf[:batch * sk, heads * d:2 * heads * d],
                       buf[:batch * sk, 2 * heads * d:3 * heads * d])
            scale = 0.37 if (sq, sk) == (129, kv + 1) else None
            y = lib.attention(q, k, v, batch, heads, sq, sk, d=d, scale=scale)
            assert torch.equal(y, lib.attention(q, k, v, batch, heads, sq, sk, d=d, scale=scale))
            sc = d ** -0.5 if scale is None else scale
            w, wl, wt = OR.attention_check(q, k, v, y, batch, heads, sq, sk, d, sc, kv_tile=kv)
            assert w <= 1.0, (d, sq, sk, w)
            # (with one key, leaving it out leaves nothing to compare)
            assert (sk == 1 or wl > 1.0) and (wt is None or wt > 1.0), (d, sq, sk, wl, wt)
    sq, sk = 129, kv + 1
    buf = torch.randn(batch * max(sq, sk), 3 * heads * d, generator=g, device="cuda").half()
    q, k, v = buf[:batch * sq, :heads * d], buf[:batch * sk, heads * d:2 * heads * d], buf[:batch * sk, 2 * heads * d:]
    mask = torch.full((batch, sk), float("-inf"), device="cuda")
    mask[0, 3], mask[1, sk - 2] = 0.5, -2.0
    y = lib.attention(q, k, v, batch, heads, sq, sk, d=d, mask=mask)
    w = OR.attention_check(q, k, v, y, batch, heads, sq, sk, d, d ** -0.5, mask=mask, kv_tile=kv, probes=False)[0]
    assert w <= 1.0, (d, "mask", w)
    for b, j in ((0, 3), (1, sk - 2)):  # every row is that key's value
        assert torch.equal(y[b * sq:(b + 1) * sq], v[b * sk + j][None].expand(sq, -1))


@pytest.mark.parametrize("dt", [F16, F32])
def test_image_postprocess_exact(cuda_lib, dt):
    """c_pad = 8 > c = 3, inputs well outside [-1, 1]: the fp32 image is exact, u8 is round(255 x image) exactly."""
    lib = cuda_lib
    g = torch.Generator(device="cuda").manual_seed(5)
    x = (2.5 * torch.randn(2, 33, 17, 8, generator=g, device="cuda")).to(dt)
    x[0, 0, 0, :3] = torch.tensor([0.0, -1.0, 1.0])
    img, u8 = lib.image_postprocess(x, c=3, want_u8=True)
    ref = OR.image_postprocess(x, 3)
    assert torch.equal(img, ref)
    assert torch.equal(u8, OR.to_u8(ref))
