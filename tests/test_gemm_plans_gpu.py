"""GPU tests of every launchable GEMM / convolution kernel instantiation (the forced-plan table of gemm_plan_cases.py)
against an fp64 reference of the same launch.

Reference.  Computed in fp64 on the device from the fp16 inputs the kernel reads: a convolution is the explicit sum over
its nine shifted taps (the taps' input windows side by side as one [M, 9 * Cin] operand, the folded shortcut's sources
appended), GroupNorm / LayerNorm / SiLU / GELU (erf) / quick-GELU / GEGLU are applied from their definitions, with the
normalisation statistics taken from the operand itself (never from the sums handed to the kernel).

Tolerance.  Per output element, |got - ref| <= r_out * |ref| + tau * B, with B the same computation on magnitudes:
B = |A| . |W|^T + |bias| + |residual|.
  * r_out = 2^-10 for fp16 output (round to nearest is within 2^-11 relative; a factor 2 of headroom); 0 for fp32
    output.  bf16 output (the bf16 VAEs): r_out = 2^-7 and tau * B charged (1 + r_out) times, the rounded fp32 value
    being itself tau * B off (test_vae_bf16_gpu.py derives both).  The staged epilogue rounds acc + bias to fp16
    before it adds the residual, so there the rounding of that intermediate is charged too: r_out * (|ref| + |pre|).
  * tau = 2^-14 for fp16 operands: products are exact in fp32 and the wgmma accumulation and the split-K / cluster
    reductions add fp32 rounding of ~2^-24 per addition; over K <= 11520 that is far below 2^-14 * sum |a w| for
    random-signed errors (a worst-case 2^-24 * K bound would reach 2^-10 only if every error had the same sign).
  * tau = 2^-11 where the kernel normalises its own operand (GroupNorm in the halo loader, the LayerNorm fold): the
    normalised operand is rounded to fp16 (2^-11 relative) and SiLU uses tanh.approx (2^-11 relative on the sigmoid),
    both relative to the normalised value, so for those cases |A| in B is the normalised operand before SiLU.
  * An activation f is Lipschitz with |f'| <= 1.13 (SiLU 1.100, GELU 1.129, quick-GELU 1.100): B becomes 1.13 * B.
    GEGLU a * gelu(g): B = |gelu(g)| * B_a + 1.13 * |a| * B_g.
One set of constants for every width and variant.

Sensitivity.  For every case the tolerance must reject the reference with one 64-channel k-block left out (the first
one, and the last, ragged one): a bound too loose to see a missing k-block fails the test instead of passing it.

Statistics outputs (rowstats, column stats) are checked against fp64 sums of the kernel's own fp16 output within
2^-14 * sum |o| (resp. sum o^2) + 1e-6: fp32 sums of a few hundred terms per partial.  Every case runs twice and must be
bit-identical (split-K reductions, cluster reductions, statistics tickets)."""
import os
import sys
import time

import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import gemm_plan_cases as G  # noqa: E402
import model_cases as MC  # noqa: E402

pytestmark = pytest.mark.gpu

R_OUT_F16 = 2.0 ** -10
R_OUT_BF16 = 2.0 ** -7
TAU = 2.0 ** -14
TAU_NORM = 2.0 ** -11
ACT_LIP = 1.13
STAT_REL = 2.0 ** -14
GN_GROUPS = 32


def _rand(g, *shape, scale=1.0, shift=0.0):
    return (torch.randn(*shape, generator=g, device="cuda") * scale + shift).half()


def _chan_sums(x):  # NHWC fp16 -> [n, c, 2] (sum, sum of squares), fp64 -> fp32
    xf = x.double().reshape(x.shape[0], -1, x.shape[-1])
    return torch.stack([xf.sum(1), (xf * xf).sum(1)], -1).float().contiguous()


def _inputs(c, seed=0):
    g = torch.Generator(device="cuda").manual_seed(1000 + seed)
    t = {}
    n, c0, c1 = c["n"], c["c0"], c["c1"]
    cin = c0 + c1
    if c["op"] == "linear":
        m = c["m"]
        shift = 0.5 if c["ln"] else 0.0
        t["x"] = _rand(g, m, c0, shift=shift)
        t["x1"] = _rand(g, m, c1, shift=shift) if c1 else None
        t["w"] = _rand(g, n, cin, scale=cin ** -0.5)
    else:
        nb, h, w = c["n_img"], c["h"], c["w"]
        shift = 0.3 if c["gn"] else 0.0
        t["x"] = _rand(g, nb, h, w, c0, shift=shift)
        t["x1"] = _rand(g, nb, h, w, c1, scale=1.7) if c1 else None
        if c["taps"] == 1:
            t["w"] = _rand(g, n, cin, scale=cin ** -0.5)
        else:
            wt = _rand(g, n, 3, 3, cin, scale=(9 * cin) ** -0.5)  # OHWI
            w2 = wt.reshape(n, 9 * cin)
            ho, wo = G.out_hw(c)
            t["s0"] = _rand(g, nb, ho, wo, c["c2"]) if c["c2"] else None
            t["s1"] = _rand(g, nb, ho, wo, c["c3"]) if c["c3"] else None
            if c["c2"]:
                ws = _rand(g, n, c["c2"] + c["c3"], scale=(c["c2"] + c["c3"]) ** -0.5)
                w2 = torch.cat([w2, ws], 1)
            t["w"] = w2.contiguous()
        if c["gn"]:
            t["gamma"] = (1.0 + 0.2 * torch.randn(cin, generator=g, device="cuda")).contiguous()
            t["beta"] = (0.1 * torch.randn(cin, generator=g, device="cuda")).contiguous()
            t["gn_groups"], t["gn_eps"] = GN_GROUPS, 1e-5
    m = G.rows(c)
    n_store = n // 2 if c["geglu"] else n
    t["bias"], t["bias_rows"], t["bias_stride"] = None, 0, 0
    if c["bias"] == "vec":
        t["bias"] = torch.randn(n, generator=g, device="cuda")
    elif c["bias"] == "img":
        rpi = G.rows_per_image(c)
        table = torch.randn((m + rpi - 1) // rpi, n + 32, generator=g, device="cuda")  # strided per-image table
        t["bias"], t["bias_rows"], t["bias_stride"] = table[:, 16:], rpi, n + 32
    t["res"] = None
    if c["residual"]:
        t["res"] = _rand(g, m, n_store) if c["op"] == "linear" else _rand(g, *t["x"].shape[:1], *G.out_hw(c), n_store)
    t["ln"] = None
    if c["ln"]:
        xf = t["x"].double()
        stat = torch.stack([xf.sum(1), (xf * xf).sum(1)], -1).float()[None].contiguous()
        t["ln"] = dict(stat=stat, parts=1, wg=t["w"].double().sum(1).float().contiguous(), eps=1e-5)
    return t


def _launch(lib, c, t):
    """The case's launch; returns (output, column statistics or None, row statistics or None)."""
    st = {} if c["stats"] else None
    rs = {} if c["rowstats"] else None
    out_dtype = torch.float32 if c["f32"] else torch.float16
    common = dict(out_dtype=out_dtype, split_k=c["split_k"], block_n=c["block_n"], bias_rows=t["bias_rows"],
                  bias_stride=t["bias_stride"], act=c["act"], stats=st, rowstats=rs, static_w=c["static_w"])
    if c["op"] == "linear":
        out = lib.linear(t["x"], t["w"], t["bias"], t["res"], x1=t["x1"], geglu=c["geglu"], ln=t["ln"], cs_hw=c["cs_hw"],
                         **common)
    else:
        gn = None
        if c["gn"]:
            gn = dict(chan0=_chan_sums(t["x"]), chan1=None if t["x1"] is None else _chan_sums(t["x1"]), gamma=t["gamma"],
                      beta=t["beta"], groups=t["gn_groups"], eps=t["gn_eps"], silu=c["silu"])
        shortcut = (t["s0"], t["s1"]) if c["c2"] else None
        out = lib.conv3x3(t["x"], t["w"], t["bias"], t["res"], x1=t["x1"], stride=c["stride"], pad_after_only=c["pad_after"],
                          halo=c["halo"], gn=gn, upsample=c["upsample"], taps=c["taps"], shortcut=shortcut, **common)
    return out, (st or {}).get("chan"), (rs or {}).get("rows")


def _group_norm(x, groups, gamma, beta, eps):  # NHWC fp64, from the definition
    n, h, w, ch = x.shape
    xg = x.reshape(n, h * w, groups, ch // groups)
    mu = xg.mean(dim=(1, 3), keepdim=True)
    var = ((xg - mu) ** 2).mean(dim=(1, 3), keepdim=True)
    y = ((xg - mu) / torch.sqrt(var + eps)).reshape(n, h, w, ch)
    return y * gamma.double() + beta.double()


def _pad(x, pad_lo, pad_hi):
    n, h, w, ch = x.shape
    xp = torch.zeros(n, h + pad_lo + pad_hi, w + pad_lo + pad_hi, ch, dtype=x.dtype, device=x.device)
    xp[:, pad_lo:pad_lo + h, pad_lo:pad_lo + w] = x
    return xp


def _taps_band(xp, stride, y0, y1, wo):
    """Padded NHWC image [h', w', c] -> the operand rows of output rows y0 <= y < y1, [(y1 - y0) * wo, 9 * c]: the
    input window of each of the nine taps, tap-major (OHWI order)."""
    cols = [xp[ty + stride * y0:ty + stride * (y1 - 1) + 1:stride, tx:tx + stride * (wo - 1) + 1:stride]
            for ty in range(3) for tx in range(3)]
    return torch.cat(cols, -1).reshape((y1 - y0) * wo, 9 * xp.shape[-1])


def _row_chunks(m, k, unit, per_image, elems=1 << 26):
    """[r0, r1) ranges covering m operand rows, each a multiple of `unit` rows inside one block of `per_image` rows,
    with at most ~elems operand elements (fp64: 512 MB) so that the 1024^2 maps' references fit beside the model."""
    step = max(unit, elems // max(1, k) // unit * unit)
    return [(r0, min(i0 + per_image, r0 + step)) for i0 in range(0, m, per_image)
            for r0 in range(i0, i0 + per_image, step)]


def _chunks(lo, ch):
    return [(lo + j, lo + min(j + 64, ch)) for j in range(0, ch, 64)]


def _operands(c, t):
    """(rows, W, k-blocks, chunks): rows(r0, r1) -> (A, |A| for the bound), rows [r0, r1) of the fp64 operand [M, K];
    the weights [N, K]; the column range of each 64-channel k-block of the kernel's main loop; the row ranges
    (_row_chunks) to evaluate the reference in."""
    c0, c1 = c["c0"], c["c1"]
    cin = c0 + c1
    x = t["x"].double() if t["x1"] is None else torch.cat([t["x"], t["x1"]], -1).double()
    mag = None
    if c["ln"]:
        mu = x.mean(-1, keepdim=True)
        x = (x - mu) / torch.sqrt(((x - mu) ** 2).mean(-1, keepdim=True) + t["ln"].get("eps", 1e-5))
    if c["gn"]:
        x = _group_norm(x, t["gn_groups"], t["gamma"], t["beta"], t["gn_eps"])
        mag = x.abs()
        if c["silu"]:
            x = x * torch.sigmoid(x)
    mag = x.abs() if mag is None else mag
    if c["upsample"]:
        x = x.repeat_interleave(2, 1).repeat_interleave(2, 2)
        mag = mag.repeat_interleave(2, 1).repeat_interleave(2, 2)
    per_tap = _chunks(0, c0) + _chunks(c0, c1)
    w = t["w"].double()
    if c["op"] == "linear" or c["taps"] == 1:
        a, am = x.reshape(-1, cin), mag.reshape(-1, cin)
        m = a.shape[0]
        return (lambda r0, r1: (a[r0:r1], am[r0:r1])), w, per_tap, _row_chunks(m, cin, 1, m)
    pad = (0, 1) if c["pad_after"] else (1, 1)
    xp, mp = _pad(x, *pad), _pad(mag, *pad)
    stride = c["stride"]
    ho, wo = x.shape[1] // stride, x.shape[2] // stride
    blocks = [(tap * cin + lo, tap * cin + hi) for tap in range(9) for lo, hi in per_tap]
    s = None
    if c["c2"]:
        s = t["s0"].double() if t["s1"] is None else torch.cat([t["s0"], t["s1"]], -1).double()
        s = s.reshape(x.shape[0] * ho * wo, -1)
        blocks += _chunks(9 * cin, c["c2"]) + _chunks(9 * cin + c["c2"], c["c3"])

    def rows(r0, r1):  # whole output rows of one image (_row_chunks with unit wo, per_image ho * wo)
        img, y0 = divmod(r0 // wo, ho)
        y1 = y0 + (r1 - r0) // wo
        a, am = _taps_band(xp[img], stride, y0, y1, wo), _taps_band(mp[img], stride, y0, y1, wo)
        if s is not None:
            a, am = torch.cat([a, s[r0:r1]], 1), torch.cat([am, s[r0:r1].abs()], 1)
        return a, am

    return rows, w, blocks, _row_chunks(x.shape[0] * ho * wo, w.shape[1], wo, ho * wo)


def _gelu(x):
    return 0.5 * x * (1.0 + torch.special.erf(x * 2.0 ** -0.5))


def _epilogue(c, t, acc, bound, r0=0):
    """fp64 epilogue of the launch's rows r0 <= r < r0 + len(acc): (ref, B, the value before the residual)."""
    m = acc.shape[0]
    y, b = acc, bound
    if t["bias"] is not None:
        bias = t["bias"].double()
        if t["bias_rows"]:
            bias = bias[torch.arange(r0, r0 + m, device=acc.device) // t["bias_rows"], : c["n"]]
        y, b = y + bias, b + bias.abs()
    if c["act"]:
        y = {1: lambda v: v * torch.sigmoid(v), 2: _gelu, 3: lambda v: v * torch.sigmoid(1.702 * v)}[c["act"]](y)
        b = ACT_LIP * b
    if c["geglu"]:
        va, gate = y[:, 0::2], y[:, 1::2]
        y, b = va * _gelu(gate), _gelu(gate).abs() * b[:, 0::2] + ACT_LIP * va.abs() * b[:, 1::2]
    pre = y
    if t["res"] is not None:
        r = t["res"].reshape(-1, y.shape[1])[r0:r0 + m].double()
        y, b = y + r, b + r.abs()
    return y, b, pre


def _tolerance(c, plan, ref, bound, pre, bf16=False):
    tau = TAU_NORM if (c["gn"] or c["ln"]) else TAU
    if c["f32"]:
        return tau * bound
    staged = plan["variant"] == 5 or plan.get("halo_kind") == 0
    scale = ref.abs() + (pre.abs() if staged and c["residual"] else 0.0)
    if bf16:
        return R_OUT_BF16 * scale + (1.0 + R_OUT_BF16) * tau * bound
    return R_OUT_F16 * scale + tau * bound


def _plan(lib, c):
    return G.parse_plan(lib.describe_plan(**G.describe_kwargs(c)))


def _check(what, c, t, plan, out, chan, rows):
    """Compare one launch's outputs with the fp64 reference, a band of rows at a time; returns the worst err / tol."""
    a_rows, w, blocks, chunks = _operands(c, t)
    bf16 = t.get("bf16", False)
    wt, wabs = w.t(), w.abs().t()
    got_all = out.double().reshape(chunks[-1][1], -1)
    worst = 0.0
    seen = {"first": False, "last": False}
    for r0, r1 in chunks:
        a, am = a_rows(r0, r1)
        acc = a @ wt
        bound0 = am @ wabs
        ref, bound, pre = _epilogue(c, t, acc, bound0, r0)
        tol = _tolerance(c, plan, ref, bound, pre, bf16)
        got = got_all[r0:r1]
        err = (got - ref).abs()
        bad = err > tol
        worst = max(worst, (err / tol).max().item())
        if bad.any():
            idx = torch.nonzero(bad)
            r, col = idx[0].tolist()
            raise AssertionError(f"{what} ({plan}): {int(bad.sum())}/{bad.numel()} elements of rows [{r0}, {r1}) out of "
                                 f"tolerance, worst err/tol {(err / tol).max().item():.3g}; rows "
                                 f"{sorted(set((idx[:, 0] + r0).tolist()))[:8]}, columns "
                                 f"{sorted(set(idx[:, 1].tolist()))[:8]}; first at ({r0 + r}, {col}): got "
                                 f"{got[r, col].item():.6g} ref {ref[r, col].item():.6g} tol {tol[r, col].item():.3g}")
        # the bound must see one missing 64-channel k-block: the first one and the last (ragged) one
        for which, (lo, hi) in (("first", blocks[0]), ("last", blocks[-1])):
            if not seen[which]:
                miss = _epilogue(c, t, acc - a[:, lo:hi] @ w[:, lo:hi].t(), bound0, r0)[0]
                seen[which] = bool(((miss - ref).abs() > tol).any())
    for which, (lo, hi) in (("first", blocks[0]), ("last", blocks[-1])):
        assert seen[which], f"{what}: tolerance cannot see the {which} k-block [{lo}, {hi}) missing"

    if rows is not None:
        o = got_all
        s = rows.double().sum(0)
        assert ((s[:, 0] - o.sum(1)).abs() <= STAT_REL * o.abs().sum(1) + 1e-6).all(), f"{what}: row sums"
        assert ((s[:, 1] - (o * o).sum(1)).abs() <= STAT_REL * (o * o).sum(1) + 1e-6).all(), f"{what}: row sums of squares"
    if chan is not None:
        o = out.double().reshape(chan.shape[0], -1, out.shape[-1])
        ref_s, ref_q = o.sum(1), (o * o).sum(1)
        assert ((chan[..., 0].double() - ref_s).abs() <= STAT_REL * o.abs().sum(1) + 1e-6).all(), f"{what}: column sums"
        assert ((chan[..., 1].double() - ref_q).abs() <= STAT_REL * ref_q + 1e-6).all(), f"{what}: column sums of squares"
    return worst


@pytest.mark.parametrize("name", [c["name"] for c in G.CASES])
def test_forced_plan_matches_fp64_reference(cuda_lib, monkeypatch, name):
    lib = cuda_lib
    c = G.CASES_BY_NAME[name]
    for k in ("B200SD_CLUSTER_SPLITK", "B200SD_STAGED"):
        monkeypatch.delenv(k, raising=False)
    for k, v in c["env"].items():
        monkeypatch.setenv(k, v)
    plan = _plan(lib, c)
    assert {k: plan.get(k) for k in c["expect"]} == c["expect"], plan

    t = _inputs(c)
    out, chan, rows = _launch(lib, c, t)
    out2, chan2, rows2 = _launch(lib, c, t)
    torch.cuda.synchronize()
    assert torch.equal(out, out2), f"{name}: second identical call differs"
    assert (chan is None or torch.equal(chan, chan2)) and (rows is None or torch.equal(rows, rows2)), name
    _check(name, c, t, plan, out, chan, rows)


# ---------------------------------------------------------------------------------------------------------------------
# Every GEMM / convolution launch of one eager forward of the shipped models, checked against the fp64 reference of that
# launch on the live activations (inputs cloned before the launch, so an output that aliases an input cannot hide an
# error), with the same tolerance and the same k-block self-check as above.
# ---------------------------------------------------------------------------------------------------------------------
def _clone(v):
    return None if v is None else v.clone()


def _bias_table(bias, n, bias_rows, bias_stride, m):
    """The bias operand as the kernel reads it: a vector of n, or one row of n per image at bias_stride."""
    if bias is None:
        return None
    if not bias_rows:
        return bias.reshape(-1)[:n].clone()
    rows = (m + bias_rows - 1) // bias_rows
    return bias.as_strided((rows, n), (bias_stride or n, 1), bias.storage_offset()).clone()


class _Replay:
    """Wraps lib.linear / lib.conv3x3: every call runs as usual, then is compared with its reference."""

    def __init__(self, lib, model):
        self.lib, self.model = lib, model
        self.linear0, self.conv0 = lib.linear, lib.conv3x3
        self.plans = {}  # distinct plan -> (calls, worst err / tol)

    def _record(self, c, t, out, st, rs):
        c["stats"] = st is not None and "chan" in st
        t["bf16"] = t["x"].dtype == torch.bfloat16
        plan = G.parse_plan(self.lib.describe_plan(**G.describe_kwargs(c), bf16=t["bf16"]))
        torch.cuda.synchronize()
        kind = "linear" if c["op"] == "linear" else ("conv1x1" if c["taps"] == 1 else "conv3x3")
        k = c["c0"] + c["c1"]
        if kind == "conv3x3":
            k = 9 * k + c["c2"] + c["c3"]
        what = f"{self.model} {kind} M={G.rows(c)} N={c['n']} K={k}"
        worst = _check(what, c, t, plan, out, None if st is None else st.get("chan"), None if rs is None else rs.get("rows"))
        key = (kind, G.rows(c), c["n"], k, plan["variant"], plan["block_n"], plan["splits"], plan["cluster"],
               plan["halo_kind"], c["gn"])
        calls, w0 = self.plans.get(key, (0, 0.0))
        self.plans[key] = (calls + 1, max(w0, worst))

    def linear(self, x, wgt, bias=None, residual=None, *, x1=None, geglu=False, out_dtype=None, split_k=0,
               block_n=0, bias_rows=0, bias_stride=0, out=None, static_w=False, act=0, ln=None, stats=None, cs_hw=0,
               rowstats=None):
        m, n = x.shape[0], wgt.shape[0]
        f32 = (out.dtype if out is not None else out_dtype) == torch.float32
        c = G.case("replay", "linear", {}, m=m, n=n, c0=x.shape[-1], c1=0 if x1 is None else x1.shape[-1],
                   bias=None if bias is None else ("img" if bias_rows else "vec"), bias_rows=bias_rows,
                   residual=residual is not None, geglu=geglu, act=act, f32=f32, ln=ln is not None,
                   rowstats=rowstats is not None, cs_hw=cs_hw, block_n=block_n, split_k=split_k, static_w=static_w)
        t = dict(x=x.clone(), x1=_clone(x1), w=wgt.clone(), res=_clone(residual), ln=None if ln is None else dict(ln),
                 bias=_bias_table(bias, n, bias_rows, bias_stride, m), bias_rows=bias_rows)
        y = self.linear0(x, wgt, bias, residual, x1=x1, geglu=geglu, out_dtype=out_dtype, split_k=split_k,
                         block_n=block_n, bias_rows=bias_rows, bias_stride=bias_stride, out=out, static_w=static_w,
                         act=act, ln=ln, stats=stats, cs_hw=cs_hw, rowstats=rowstats)
        self._record(c, t, y, stats, rowstats)
        return y

    def conv3x3(self, x, wgt, bias=None, residual=None, *, x1=None, stride=1, out_dtype=None, split_k=0,
                block_n=0, bias_rows=0, bias_stride=0, out=None, act=0, static_w=True, pad_after_only=False,
                halo=False, gn=None, upsample=False, stats=None, rowstats=None, taps=9, shortcut=None):
        nimg, h, w, c0 = x.shape
        n = wgt.shape[0]
        s0, s1 = shortcut if shortcut is not None else (None, None)
        f32 = (out.dtype if out is not None else out_dtype) == torch.float32
        c = G.case("replay", "conv", {}, n_img=nimg, h=h, w=w, c0=c0, n=n, c1=0 if x1 is None else x1.shape[-1],
                   c2=0 if s0 is None else s0.shape[-1], c3=0 if s1 is None else s1.shape[-1], stride=stride,
                   pad_after=pad_after_only, bias=None if bias is None else ("img" if bias_rows else "vec"),
                   bias_rows=bias_rows, residual=residual is not None, act=act, f32=f32, rowstats=rowstats is not None,
                   halo=int(halo), gn=gn is not None, silu=bool(gn and gn["silu"]), upsample=upsample, taps=taps,
                   block_n=block_n, split_k=split_k, static_w=static_w)
        t = dict(x=x.clone(), x1=_clone(x1), w=wgt.clone(), res=_clone(residual), s0=_clone(s0), s1=_clone(s1),
                 bias=_bias_table(bias, n, bias_rows, bias_stride, G.rows(c)), bias_rows=bias_rows, ln=None)
        if gn is not None:
            t.update(gamma=gn["gamma"].clone(), beta=gn["beta"].clone(), gn_groups=int(gn["groups"]), gn_eps=float(gn["eps"]))
        y = self.conv0(x, wgt, bias, residual, x1=x1, stride=stride, out_dtype=out_dtype, split_k=split_k, block_n=block_n,
                       bias_rows=bias_rows, bias_stride=bias_stride, out=out, act=act, static_w=static_w,
                       pad_after_only=pad_after_only, halo=halo, gn=gn, upsample=upsample, stats=stats,
                       rowstats=rowstats, taps=taps, shortcut=shortcut)
        self._record(c, t, y, stats, rowstats)
        return y

    def report(self):
        lines = [f"{self.model}: {sum(v[0] for v in self.plans.values())} launches, {len(self.plans)} distinct plans"]
        for (kind, m, n, k, var, bn, sp, cl, hk, gn), (calls, worst) in sorted(self.plans.items(), key=str):
            ker = (f"halo kind {hk}" + (" + GN" if gn else "")) if var < 0 else G.VARIANTS[var]
            lines.append(f"  {kind:8s} M={m:6d} N={n:5d} K={k:6d}  {ker:16s} width {bn:3d} splits {sp} cluster {cl}"
                         f"  x{calls:<3d} worst err/tol {worst:.3f}")
        return "\n".join(lines)


MODELS = MC.SHIPPED + ["sd21_b2_fused", "sd21_b2_halo_tma", "sd15_512x768_b2_fused", "sd15_512x768_b2_halo_tma"]


@pytest.mark.parametrize("name", MODELS)
def test_model_launches_match_fp64_reference(cuda_lib, monkeypatch, name):
    """Every model of model_cases.SHIPPED from random-init weights (the bf16 VAEs against the bf16 output bound); SD-2.1
    and SD-1.5 at 512x768 (halo windows and the cs_hw tile-to-image mapping on a non-square map) twice more with the
    opt-in halo convolutions: B200SD_FUSED=1 (GroupNorm + SiLU in the halo kernel's operand path,
    kinds 0 / 1) and B200SD_HALO_TMA=1024 (plain convolutions on maps of >= 1024 pixels with TMA patches, kind 2).
    Under B200SD_FUSED=1 every convolution behind a GroupNorm takes the GroupNorm-fused kernel, so B200SD_HALO_TMA has
    nothing left to take there: kind 2 needs the run of its own.  Prints one line per distinct plan and the wall time
    of the build, forward and checks (run with -s); GEMM_PLANS.md holds these tables as measured on an H100."""
    lib = cuda_lib
    for k in ("B200SD_CLUSTER_SPLITK", "B200SD_STAGED", "B200SD_FUSED", "B200SD_HALO_TMA"):
        monkeypatch.delenv(k, raising=False)
    if name.endswith("_fused"):
        monkeypatch.setenv("B200SD_FUSED", "1")
        monkeypatch.setenv("B200SD_HALO_TMA", "1024")
    if name.endswith("_halo_tma"):
        monkeypatch.setenv("B200SD_HALO_TMA", "1024")
    t0 = time.perf_counter()
    m = MC.build(name)
    rep = _Replay(lib, name)
    monkeypatch.setattr(lib, "linear", rep.linear)
    monkeypatch.setattr(lib, "conv3x3", rep.conv3x3)
    m(**MC.model_inputs(m, seed=9))
    torch.cuda.synchronize()
    print(f"\n{rep.report()}\n  wall time {time.perf_counter() - t0:.1f} s")
    assert rep.plans, f"{name}: no GEMM / convolution launch was seen"
    halo = {(key[8], key[9]) for key in rep.plans}  # (halo_kind, GroupNorm fused)
    if name.endswith("_fused"):  # the opt-in paths this run exists for were taken
        assert (0, True) in halo and any(kind == 1 for kind, _ in halo), f"{name}: halo kinds seen {sorted(halo)}"
    elif name.endswith("_halo_tma"):
        assert (2, False) in halo, f"{name}: halo kinds seen {sorted(halo)}"
