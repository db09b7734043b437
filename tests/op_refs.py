"""fp64 references, error bounds and sensitivity probes of the attention, normalisation and elementwise kernels (see
test_op_launches_gpu.py for the derivation of every bound).  Device-agnostic: the same functions run on CPU tensors in
test_op_refs.py, where the bounds are shown to accept the exact reference and to reject each perturbed one.

Every check returns (ref, tol) as fp64 tensors shaped like the kernel's output; a launch passes when
|got - ref| <= tol everywhere, and a bound is tight enough when a perturbed reference leaves it somewhere."""
import torch

# unit roundoff of the output type, times 2 (the GEMM tests' convention): round to nearest is within half an ulp
R_OUT = {torch.float16: 2.0 ** -10, torch.bfloat16: 2.0 ** -7, torch.float32: 0.0}
# absolute floor: half the smallest fp16 subnormal (bf16 and fp32 keep fp32's exponent range)
TINY = {torch.float16: 2.0 ** -25, torch.bfloat16: 2.0 ** -127, torch.float32: 2.0 ** -127}
ACT_LIP = 1.13          # |SiLU'| <= 1.100 (the GEMM tests' one constant for every activation)
SILU_REL = 2.0 ** -19   # __expf (ex2.approx of a rounded product) + __fdividef: relative error of silu_f
E_SUM = 2.0 ** -18      # relative error of a kernel's own fp32 statistics sums (GroupNorm, LayerNorm, softmax)
E_PRODUCER = 2.0 ** -14  # relative error of a producer's per-channel sums (asserted by test_gemm_plans_gpu.py)
K_STAT = 8.0            # attention: multiple of the random-walk error of the fp16 probabilities
F32 = 2.0 ** -24


def silu(y):
    return y * torch.sigmoid(y)


def worst(got, ref, tol):
    """max err / tol (0 for an empty tensor)."""
    if ref.numel() == 0:
        return 0.0
    return float(((got.double() - ref).abs() / tol).max())


def rejects(alt, ref, tol):
    """True if the perturbed reference `alt` leaves the bound around `ref` somewhere."""
    return bool(((alt - ref).abs() > tol).any())


# ---- GroupNorm ------------------------------------------------------------------------------------------------------
def gn_stats(x, groups, shift=0, px=None):
    """x fp64 [n, hw, C] -> per (image, group) mean and (biased) variance.  Perturbations: shift moves every group's
    channel range by `shift` channels (cyclically); px restricts the statistics to that pixel slice."""
    n, hw, c = x.shape
    xs = torch.roll(x, -shift, dims=-1) if shift else x
    if px is not None:
        xs = xs[:, px]
    xg = xs.reshape(n, xs.shape[1], groups, c // groups)
    mu = xg.mean(dim=(1, 3))
    return mu, ((xg - mu[:, None, :, None]) ** 2).mean(dim=(1, 3))


def group_norm(x, gamma, beta, groups, eps, silu_, out_dtype, e_sum=E_SUM, stats=None):
    """x fp64 [n, hw, C] -> (ref, tol).  stats: (mean, var) [n, groups] to normalise with instead of the true ones (the
    perturbed reference of a sensitivity probe; tol is still the true one's)."""
    n, hw, c = x.shape
    cpg = c // groups
    mu, var = gn_stats(x, groups)
    sd = torch.sqrt(var + eps)
    rho = (mu.abs() / sd).repeat_interleave(cpg, 1)[:, None]
    g, b = gamma.double(), beta.double()

    def apply(m, v):
        xh = (x - m.repeat_interleave(cpg, 1)[:, None]) / torch.sqrt(v + eps).repeat_interleave(cpg, 1)[:, None]
        y = xh * g + b
        return (silu(y) if silu_ else y), xh

    ref, xh = apply(mu, var)
    # one-pass variance: sums carry e_sum relative error, so var (+eps) is off by e_sum (mu^2 + var) -> relative
    # e_sum (1 + rho^2) and rstd by half that; the mean by e_sum mean|x| <= e_sum (|mu| + sigma), i.e. e_sum (1 + rho)
    # in units of sigma.  The apply's fp32 FMA with shift beta - mu * scale adds ~2^-22 (|x_hat| + rho) |gamma| + |beta|.
    bound = g.abs() * (xh.abs() * 0.5 * (1 + rho ** 2) + 1 + rho) * e_sum + 2.0 ** -22 * b.abs()
    r = R_OUT[out_dtype] + (SILU_REL if silu_ else 0.0)
    tol = r * ref.abs() + TINY[out_dtype] + (ACT_LIP if silu_ else 1.0) * bound
    if stats is not None:
        ref = apply(*stats)[0]
    return ref, tol


# ---- LayerNorm (two-pass in registers) ------------------------------------------------------------------------------
def layer_norm(x, gamma, beta, eps, shift=0):
    """x fp64 [rows, C] -> (ref, tol).  shift: the perturbed reference whose row statistics are taken over channels
    [shift, C + shift) of the flattened tensor (every row boundary moved by `shift` channels)."""
    rows, c = x.shape
    xs = torch.roll(x.reshape(-1), -shift).reshape(rows, c) if shift else x
    mu = xs.mean(-1, keepdim=True)
    var = ((xs - mu) ** 2).mean(-1, keepdim=True)
    xh = (x - mu) / torch.sqrt(var + eps)
    ref = xh * gamma.double() + beta.double()
    if shift:
        return ref, None
    mu0, sd0 = mu, torch.sqrt(var + eps)
    rho = mu0.abs() / sd0
    # two-pass: the mean is off by E (|mu| + sigma), which enters var only squared: relative E + E^2 (1 + rho)^2
    bound = gamma.double().abs() * (xh.abs() * 0.5 * (E_SUM + (E_SUM * (1 + rho)) ** 2) + E_SUM * (1 + rho))
    tol = R_OUT[torch.float16] * ref.abs() + TINY[torch.float16] + bound + 2.0 ** -22 * beta.double().abs()
    return ref, tol


# ---- row softmax ----------------------------------------------------------------------------------------------------
def softmax_rows(s, scale, out_dtype, drop_last=False):
    """fp32 scores [rows, cols] -> (ref, tol).  Kernel: z = s * (scale * log2 e) in fp32, m = max z, exp2f(z - m) summed
    in fp32, times the rounded reciprocal.  Per element, relative: output rounding; E_SUM for the sum and the reciprocal;
    the rounding of z_i and of the max shifts the exponent by 2^-24 (|z_i| + |m|) (times ln 2 < 1) and the subtraction
    by 2^-24 |z_i - m|; exp2f itself is within 2 ulp.  drop_last: the reference with its last column left out."""
    sl2 = torch.tensor(scale, dtype=torch.float32) * torch.tensor(1.4426950408889634, dtype=torch.float32)
    z = s.double() * float(sl2)
    zz = z[:, :-1] if drop_last else z
    m = zz.max(-1, keepdim=True).values
    e = torch.exp2(zz - m)
    ref = e / e.sum(-1, keepdim=True)
    if drop_last:
        ref = torch.cat([ref, torch.zeros_like(z[:, -1:])], -1)
        return ref, None
    rel = R_OUT[out_dtype] + E_SUM + F32 * (2 * z.abs() + 2 * m.abs() + 4)
    return ref, rel * ref + TINY[out_dtype]


# ---- small-M linear -------------------------------------------------------------------------------------------------
def linear_small(x, w, bias, add, act_in, act_out, drop_last_k=False):
    """fp32 x [m, k] . fp16 w [n, k]^T (+ bias + add per column), SiLU on the input / output -> (ref, tol), fp32 output.
    B = |x'| . |w|^T + |bias| + |add| (x' = silu(x) with act_in); fp32 sums of <= k products in a fixed tree: random-signed
    2^-24 per addition, 2^-20 B leaves 16x; silu_f adds SILU_REL relative on x' and on the output; ACT_LIP with act_out.
    drop_last_k: the reference without the last 8 input features (one 16-byte weight vector per lane)."""
    xd = x.double()
    if act_in:
        xd = silu(xd)
    wd = w.double()
    if drop_last_k:
        xd, wd = xd[:, :-8], wd[:, :-8]
    acc = xd @ wd.t()
    bnd = xd.abs() @ wd.abs().t() * (2.0 ** -20 + (SILU_REL if act_in else 0.0))
    for t in (bias, add):
        if t is not None:
            acc = acc + t.double()
            bnd = bnd + 2.0 ** -23 * t.double().abs()
    if act_out:
        return silu(acc), ACT_LIP * bnd + SILU_REL * silu(acc).abs()
    return acc, bnd


# ---- sinusoidal timestep embedding ----------------------------------------------------------------------------------
def timestep_embedding(t, dim, flip, freq_shift, perturb=False):
    """-> (ref, tol) [m, dim] fp32.  freq_j = exp(-ln(10^4) j / (dim / 2 - shift)) is evaluated in fp32 from three
    rounded operations and expf: relative error < 2^-18 for |ln(10^4) j / (...)| <= 9.3; the angle t * freq adds one
    rounding.  sinf / cosf are within 2 ulp of the rounded angle, so |err| <= 2^-18 |angle| + 2^-21 (|angle| <= 1000:
    < 4e-3).  perturb: the reference with the frequency index shifted by one (a wrong frequency table)."""
    half = dim // 2
    j = torch.arange(half, dtype=torch.float64, device=t.device) + (1 if perturb else 0)
    freq = torch.exp(-torch.log(torch.tensor(10000.0, dtype=torch.float64)) * j / (half - freq_shift))
    ang = t.double()[:, None] * freq.to(t.device)
    s, c = torch.sin(ang), torch.cos(ang)
    ref = torch.cat([c, s], -1) if flip else torch.cat([s, c], -1)
    tol = 2.0 ** -18 * torch.cat([ang.abs(), ang.abs()], -1) + 2.0 ** -21
    return ref, tol


# ---- VAE latent prep: post_quant_conv(z * inv_scale) ----------------------------------------------------------------
def latent_prep(z, w, b, inv_scale, c_pad, out_dtype, drop_last=False):
    """fp32 NCHW z -> (ref, tol) NHWC [n, h, w, c_pad].  fp32 products and <= 8 additions: 2^-21 B on top of the output
    rounding, B = |b| + |w| . |z * inv_scale|.  drop_last: the reference without the last input channel."""
    n, c, h, wd = z.shape
    v = (z.double() * float(torch.tensor(inv_scale, dtype=torch.float32))).permute(0, 2, 3, 1)
    wm = w.double().reshape(c, c)
    if drop_last:
        v, wm = v[..., :-1], wm[:, :-1]
    y, bnd = v @ wm.t(), v.abs() @ wm.abs().t()
    if b is not None:
        y, bnd = y + b.double(), bnd + b.double().abs()
    ref = torch.zeros(n, h, wd, c_pad, dtype=torch.float64, device=z.device)
    tol = torch.zeros_like(ref)
    ref[..., :c] = y
    tol[..., :c] = R_OUT[out_dtype] * y.abs() + 2.0 ** -21 * bnd + TINY[out_dtype]
    tol[..., c:] = TINY[out_dtype]
    return ref, tol


# ---- flash attention ------------------------------------------------------------------------------------------------
def attention_check(q, k, v, out, batch, heads, sq, sk, d, scale, mask=None, causal=False, kv_tile=128, probes=True,
                    max_elems=1 << 23):
    """Compares one attention launch with its fp64 reference, chunked over (image, head, query block) so that no
    [query block, sk] matrix exceeds max_elems.  q / k / v / out are the views the kernel read and wrote
    ([rows, >= heads * d], any row stride).  Returns (worst err / tol, worst |ref_drop_last - ref| / tol,
    worst |ref_drop_first_tile - ref| / tol or None when sk fits one K/V tile); the probe ratios are None with
    probes=False.

    Bound per output element: r_out |ref| + K_STAT R (2^-11 + (d + 2) 2^-24 S) + 2^-20 B + TINY with, over the keys j of
    the row, P the probabilities, B = P . |V|, R = sqrt(sum_j P_j^2 V_j^2) and S = max_j (scale sum_d |q_d k_jd| + |mask_j|).
    P enters the PV product rounded to fp16 (2^-11 relative each, random-signed over the keys: its effect on O is a
    random walk of size 2^-11 R, K_STAT of those being far outside its spread); the scores are fp32 sums of d exact products
    (<= (d + 2) 2^-24 S absolute, again per key); ex2.approx, the fp32 sums of P and O and the stream-K merges are within
    2^-20 of B."""
    dev = out.device
    r_out, tiny = R_OUT[torch.float16], TINY[torch.float16]
    wmax, wlast, wtile = 0.0, 0.0, 0.0
    has_tile = sk > kv_tile
    qb = max(1, min(sq, max_elems // max(1, sk)))
    for b in range(batch):
        mrow = None if mask is None else mask[b].double().to(dev)
        for h in range(heads):
            cols = slice(h * d, (h + 1) * d)
            kk = k[b * sk:(b + 1) * sk, cols].double()
            vv = v[b * sk:(b + 1) * sk, cols].double()
            va, v2 = vv.abs(), vv * vv
            for q0 in range(0, sq, qb):
                q1 = min(sq, q0 + qb)
                qq = q[b * sq + q0:b * sq + q1, cols].double()
                s = (qq @ kk.t()) * scale
                sabs = (qq.abs() @ kk.abs().t()) * scale
                if mrow is not None:
                    s = s + mrow
                    sabs = sabs + torch.where(torch.isfinite(mrow), mrow.abs(), torch.zeros_like(mrow))
                if causal:
                    vis = torch.arange(sk, device=dev)[None, :] <= torch.arange(q0, q1, device=dev)[:, None]
                    s = torch.where(vis, s, torch.full_like(s, float("-inf")))
                m = s.max(-1, keepdim=True).values
                e = torch.exp(s - m)
                l = e.sum(-1, keepdim=True)
                num = e @ vv
                ref = num / l
                bnd = (e @ va) / l
                rw = torch.sqrt((e * e) @ v2) / l
                smax = torch.where(torch.isfinite(s), sabs, torch.zeros_like(sabs)).max(-1, keepdim=True).values
                tol = r_out * ref.abs() + K_STAT * rw * (2.0 ** -11 + (d + 2) * F32 * smax) + 2.0 ** -20 * bnd + tiny
                got = out[b * sq + q0:b * sq + q1, cols].double()
                wmax = max(wmax, float(((got - ref).abs() / tol).max()))
                if not probes:
                    continue
                # the last key left out, and the first K/V tile
                el = e[:, -1:]
                alt = (num - el * vv[-1:]) / (l - el)
                wlast = max(wlast, float(torch.nan_to_num((alt - ref).abs() / tol, nan=0.0).max()))
                if has_tile:
                    et = e[:, :kv_tile]
                    alt = (num - et @ vv[:kv_tile]) / (l - et.sum(-1, keepdim=True))
                    wtile = max(wtile, float(torch.nan_to_num((alt - ref).abs() / tol, nan=0.0, posinf=1e30).max()))
    if not probes:
        return wmax, None, None
    return wmax, wlast, (wtile if has_tile else None)


# ---- image post-processing ------------------------------------------------------------------------------------------
def image_postprocess(x, c):
    """NHWC(c_pad) fp16 / fp32 -> the fp32 image clip(x / 2 + 0.5, 0, 1) of the first c channels, evaluated as the kernel
    does (x * 0.5 is exact, one fp32 rounding in the addition): the kernel's result exactly."""
    return torch.clamp(x[..., :c].float() * 0.5 + 0.5, 0.0, 1.0)


def to_u8(img):
    """diffusers' numpy_to_pil rounding: round(255 * image) (half to even), in fp32."""
    return torch.round(img * 255.0).to(torch.uint8)
