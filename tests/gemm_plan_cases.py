"""Forced-plan cases of the GEMM / convolution kernels (csrc/gemm_conv.cu), shared by test_gemm_plans.py (host: every
case plans the kernel it names, and the table reaches every kernel a launch can run) and test_gemm_plans_gpu.py (device: every
case against an fp64 reference of the same launch).

wgmma_gemm_kernel is compiled once per (epilogue variant, tile width), 6 x 8 = 48 instantiations.  A launch can reach
43 of them: variants 1..5 need block_n % 32 == 0, so width 16 always takes the generic variant 0.  The halo
convolution has kinds 0 / 1 / 2, kind 2 in a narrow and a wide (block_n > 128) instantiation.  The cost model alone
would reach only the kernels its shapes favour, so each case forces its kernel (block_n, split_k,
B200SD_CLUSTER_SPLITK=0, B200SD_STAGED=1) and names the plan it expects: a planner change that moves a case to another
kernel fails the host test instead of turning the case into a duplicate.

Shapes sit where tiled kernels break: M not a multiple of 128 (and M < 128), N not a multiple of the tile width (and
N % 16 != 0 for the generic variant), ragged 64-channel k-chunks (c0 / c1 / c2 / c3 not multiples of 64, c0 = 8)."""

WIDTHS = (256, 192, 160, 128, 96, 64, 32, 16)
VARIANTS = {0: "generic", 1: "split-K partial", 2: "GEGLU", 3: "fp32 output", 4: "plain", 5: "staged"}
GEMM_KERNELS = frozenset({(v, w) for v in range(1, 6) for w in WIDTHS[:-1]} | {(0, w) for w in WIDTHS})
HALO_KERNELS = frozenset({(0, 0), (1, 0), (2, 0), (2, 1)})  # (halo_kind, halo_wide)

NO_CLUSTER = {"B200SD_CLUSTER_SPLITK": "0"}
STAGED = {"B200SD_STAGED": "1"}


def case(name, op, expect, **kw):
    """A launch description: op "linear" (m, n, c0, c1) or "conv" (n_img, h, w input size, c0, c1, n output channels,
    stride, pad_after, folded shortcut c2 / c3, halo kind, gn, upsample, taps); bias None / "vec" / "img" (a per-image
    table, bias_rows rows per image); the fused outputs and inputs (stats, rowstats with cs_hw, ln); the forcing
    (block_n, split_k, env) and the plan fields it expects."""
    c = dict(name=name, op=op, expect=expect, m=0, n=0, c0=0, n_img=0, h=0, w=0, c1=0, c2=0, c3=0, stride=1,
             pad_after=False, bias="vec", bias_rows=0, residual=False, geglu=False, act=0, f32=False, ln=False, stats=False,
             rowstats=False, cs_hw=0, halo=0, gn=False, silu=True, upsample=False, taps=9, block_n=0, split_k=1,
             env={}, static_w=True)
    unknown = set(kw) - set(c)
    assert not unknown, unknown
    c.update(kw)
    return c


def _lin(name, expect, m, n, c0, **kw):
    return case(name, "linear", expect, m=m, n=n, c0=c0, **kw)


def _conv(name, expect, n_img, h, w, c0, n, **kw):
    return case(name, "conv", expect, n_img=n_img, h=h, w=w, c0=c0, n=n, **kw)


def _v(variant, bn, splits=1, cluster=0, **extra):
    return dict(variant=variant, block_n=bn, splits=splits, cluster=cluster, **extra)


def _h(kind, bn, **extra):
    return dict(variant=-1, halo_kind=kind, halo_wide=int(bn > 128), block_n=bn, **extra)


CASES = [
    # ---- plain (4): bias vectors, two sources, residual + row statistics on the register epilogue, convolutions ----
    _lin("plain256_lin_res_rowstats", _v(4, 256, res_smem=1), 200, 320, 520, residual=True, rowstats=True, block_n=256),
    _conv("plain192_conv8x8_bnimg2", _v(4, 192, box=(2, 8, 8)), 2, 8, 8, 72, 400, block_n=192),
    _lin("plain160_lin_two_src", _v(4, 160), 129, 336, 64, c1=32, block_n=160),
    _conv("plain128_conv24x40", _v(4, 128), 1, 24, 40, 64, 144, block_n=128),
    _lin("plain96_lin_m77_untiled", _v(4, 96), 77, 208, 1024, block_n=96, static_w=False),
    _conv("plain64_conv_stride2", _v(4, 64), 2, 16, 16, 128, 80, stride=2, block_n=64),
    _conv("plain32_conv_pad_after_only", _v(4, 32), 1, 24, 40, 64, 48, stride=2, pad_after=True, block_n=32),
    _conv("plain160_conv_in_c8", _v(4, 160), 2, 32, 32, 8, 320, bias=None, block_n=160),
    _conv("plain128_conv_two_src_temb", _v(4, 128, bias_mode=1), 2, 16, 16, 64, 128, c1=32, bias="img", block_n=128),
    _conv("plain128_conv_shortcut", _v(4, 128), 2, 8, 8, 64, 144, c2=72, c3=40, block_n=128),
    # ---- GEGLU (2): interleaved (value, gate) rows ----
    _lin("geglu256", _v(2, 256), 154, 640, 320, geglu=True, block_n=256),
    _lin("geglu192", _v(2, 192), 200, 416, 136, geglu=True, block_n=192),
    _lin("geglu160", _v(2, 160), 129, 352, 64, geglu=True, block_n=160),
    _lin("geglu128", _v(2, 128), 256, 288, 96, geglu=True, block_n=128, static_w=False),
    _lin("geglu96_m100", _v(2, 96), 100, 224, 128, geglu=True, block_n=96),
    _lin("geglu64_ln", _v(2, 64), 300, 176, 72, geglu=True, ln=True, block_n=64),
    _lin("geglu32_two_src", _v(2, 32), 154, 80, 64, c1=64, geglu=True, block_n=32),
    # ---- fp32 output (3), residual through the register path ----
    _lin("f32_256_res", _v(3, 256, res_smem=1), 200, 288, 256, residual=True, f32=True, block_n=256),
    _conv("f32_192_conv8x8", _v(3, 192), 2, 8, 8, 64, 208, f32=True, block_n=192),
    _lin("f32_160_m77", _v(3, 160), 77, 176, 520, f32=True, block_n=160),
    _conv("f32_128_conv24x40_res", _v(3, 128, res_smem=1), 1, 24, 40, 72, 144, residual=True, f32=True, block_n=128),
    _lin("f32_96_res", _v(3, 96, res_smem=1), 129, 112, 64, residual=True, f32=True, block_n=96),
    _lin("f32_64_ln", _v(3, 64), 300, 80, 128, f32=True, ln=True, block_n=64),
    _conv("f32_32_conv_stride2", _v(3, 32), 2, 8, 8, 96, 48, stride=2, f32=True, block_n=32),
    # ---- staged (5): column statistics, B200SD_STAGED=1 residual ----
    _lin("staged256_res_rowstats", _v(5, 256), 256, 320, 320, residual=True, rowstats=True, block_n=256, env=STAGED),
    _conv("staged192_conv_stats", _v(5, 192), 2, 16, 16, 128, 208, stats=True, block_n=192),
    _lin("staged160_stats_rowstats", _v(5, 160), 512, 336, 72, stats=True, cs_hw=256, rowstats=True, block_n=160),
    _conv("staged128_conv8x8_stats_temb", _v(5, 128, box=(2, 8, 8)), 2, 8, 8, 64, 144, stats=True, bias="img",
          block_n=128),
    _lin("staged96_res_m200", _v(5, 96), 200, 112, 128, residual=True, block_n=96, env=STAGED),
    _conv("staged64_conv24x40_stats_res", _v(5, 64), 1, 24, 40, 64, 80, stats=True, residual=True, block_n=64),
    _lin("staged32_stats_res", _v(5, 32), 128, 48, 64, stats=True, cs_hw=64, rowstats=True, residual=True, block_n=32),
    # ---- split-K through the fp32 workspace and the reduce kernel (1) ----
    _lin("ws256_split3", _v(1, 256, 3), 200, 288, 1280, residual=True, block_n=256, split_k=3),
    _lin("ws192_split7", _v(1, 192, 7), 129, 400, 896, residual=True, block_n=192, split_k=7),
    _lin("ws160_split2", _v(1, 160, 2), 77, 336, 520, block_n=160, split_k=2, env=NO_CLUSTER),
    _conv("ws128_conv_split2_temb_res", _v(1, 128, 2), 2, 8, 8, 320, 144, c1=72, bias="img", residual=True,
          block_n=128, split_k=2, env=NO_CLUSTER),
    _lin("ws96_split7_uneven_ragged", _v(1, 96, 7, kb_per_split=3), 154, 208, 1256, residual=True, f32=True,
         block_n=96, split_k=7),
    _lin("ws64_split3", _v(1, 64, 3), 300, 80, 1152, block_n=64, split_k=3),
    _lin("ws32_split4", _v(1, 32, 4), 100, 48, 1024, residual=True, block_n=32, split_k=4, env=NO_CLUSTER),
    # ---- split-K reduced inside a thread-block cluster (1) ----
    _lin("cl256_split2", _v(1, 256, 2, 1), 2000, 288, 1280, residual=True, block_n=256, split_k=2),
    _lin("cl192_split4", _v(1, 192, 4, 1), 129, 400, 1024, residual=True, block_n=192, split_k=4),
    _lin("cl160_split8", _v(1, 160, 8, 1), 77, 336, 2048, block_n=160, split_k=8),
    _conv("cl128_conv_split4_temb_res", _v(1, 128, 4, 1), 2, 8, 8, 320, 144, c1=72, bias="img", residual=True,
          block_n=128, split_k=4),
    _lin("cl96_split2_f32", _v(1, 96, 2, 1), 154, 208, 640, residual=True, f32=True, block_n=96, split_k=2),
    _lin("cl64_split8", _v(1, 64, 8, 1), 300, 80, 1152, block_n=64, split_k=8),
    _lin("cl32_split4", _v(1, 32, 4, 1), 100, 48, 1024, residual=True, block_n=32, split_k=4),
    # ---- generic (0): N % 16 != 0, activations, row-gathered per-image bias, fp32 output with N = 4 ----
    _lin("gen256_n260_res", _v(0, 256), 200, 260, 256, residual=True, block_n=256),
    _lin("gen192_bias_rows77", _v(0, 192, bias_mode=2), 154, 400, 256, bias="img", bias_rows=77, residual=True,
         block_n=192),
    _lin("gen160_quick_gelu", _v(0, 160), 129, 336, 64, act=3, block_n=160),
    _conv("gen128_conv4x4_bnimg8_temb", _v(0, 128, bias_mode=2, box=(4, 4, 8)), 3, 4, 4, 128, 144, bias="img",
          block_n=128),
    _lin("gen96_gelu", _v(0, 96), 77, 208, 1024, act=2, block_n=96),
    _lin("gen64_n200_res", _v(0, 64), 200, 200, 72, residual=True, block_n=64),
    _lin("gen32_silu", _v(0, 32), 154, 80, 64, act=1, block_n=32, static_w=False),
    _conv("gen16_conv_out_n4_f32", _v(0, 16), 2, 16, 16, 320, 4, f32=True, block_n=16),
    _conv("gen16_conv_out_n4_f32_split3", _v(0, 16, 3), 2, 16, 16, 320, 4, f32=True, block_n=16, split_k=3),
    _lin("gen16_n40", _v(0, 16), 129, 40, 136, residual=True, block_n=16),
    # ---- halo convolution: kind 1 (block_n 16, fp32 / narrow output) ----
    _conv("halo1_n4_f32", _h(1, 16, win=0), 1, 24, 24, 64, 4, f32=True, halo=1, block_n=16),
    _conv("halo1_window_gn", _h(1, 16, win=1), 1, 12, 96, 64, 16, halo=1, gn=True, block_n=16),
    # ---- kind 0 (loader warps, staged epilogue): GroupNorm (+SiLU), upsample, 1x1 taps, statistics, windows ----
    _conv("halo0_32_gn_two_src", _h(0, 32, win=0), 2, 12, 20, 64, 48, c1=32, halo=1, gn=True, block_n=32),
    _conv("halo0_64_upsample_window", _h(0, 64, win=1), 1, 12, 40, 64, 80, halo=1, upsample=True, block_n=64),
    _conv("halo0_96_1x1_gn_rowstats", _h(0, 96), 2, 16, 16, 128, 208, halo=1, gn=True, silu=False, taps=1,
          rowstats=True, block_n=96),
    _conv("halo0_128_window_stats_res", _h(0, 128, win=1), 1, 20, 96, 72, 144, halo=1, stats=True, residual=True,
          block_n=128),
    # ---- kind 2 (TMA patches): narrow and wide instantiations ----
    _conv("halo2_32_temb_res", _h(2, 32), 2, 8, 8, 64, 48, halo=2, bias="img", residual=True, block_n=32),
    _conv("halo2_64_window", _h(2, 64, win=1), 1, 24, 96, 96, 80, halo=2, block_n=64),
    _conv("halo2_96", _h(2, 96), 1, 16, 16, 320, 112, halo=2, block_n=96),
    _conv("halo2_128_two_src", _h(2, 128), 2, 16, 16, 64, 160, c1=72, halo=2, block_n=128),
    _conv("halo2_160_wide", _h(2, 160), 1, 16, 24, 128, 336, halo=2, block_n=160),
    _conv("halo2_192_wide", _h(2, 192), 2, 12, 12, 64, 208, halo=2, block_n=192),
    _conv("halo2_256_wide_res", _h(2, 256, win=0), 1, 16, 40, 64, 320, halo=2, residual=True, block_n=256),
]

CASES_BY_NAME = {c["name"]: c for c in CASES}
assert len(CASES_BY_NAME) == len(CASES)


def out_hw(c):
    """Output height / width of a convolution case."""
    h, w = (2 * c["h"], 2 * c["w"]) if c["upsample"] else (c["h"], c["w"])
    return h // c["stride"], w // c["stride"]


def rows(c):
    """M of the launch."""
    if c["op"] == "linear":
        return c["m"]
    ho, wo = out_hw(c)
    return c["n_img"] * ho * wo


def rows_per_image(c):
    """Rows that share one per-image bias row / one set of column statistics."""
    if c["op"] == "linear":
        return c["bias_rows"] or c["cs_hw"]
    ho, wo = out_hw(c)
    return ho * wo


def describe_kwargs(c):
    """Arguments of lib.describe_plan for the launch this case makes."""
    kw = dict(n=c["n"], c0=c["c0"], c1=c["c1"], geglu=c["geglu"], has_bias=c["bias"] is not None,
              has_residual=c["residual"], split_k=c["split_k"], block_n=c["block_n"], out_f32=c["f32"], act=c["act"],
              rowstats=c["rowstats"], stats=c["stats"], ln=c["ln"], c2=c["c2"], c3=c["c3"], halo=c["halo"],
              upsample=c["upsample"], gn=c["gn"])
    if c["bias"] == "img":
        kw["bias_rows"] = c["bias_rows"] or rows_per_image(c)
    if c["op"] == "linear":
        kw.update(mode=0, m=c["m"], cs_hw=c["cs_hw"])
    else:
        h, w = (2 * c["h"], 2 * c["w"]) if c["upsample"] else (c["h"], c["w"])
        kw.update(mode=1 if c["taps"] == 9 else 0, n_img=c["n_img"], h=h, w=w, stride=c["stride"],
                  pad_after_only=c["pad_after"], m=rows(c) if c["taps"] == 1 else 0)
    return kw


def parse_plan(s):
    """'key=value ...' of b200sd_gemm_describe_plan -> dict (box=AxBxC -> tuple)."""
    out = {}
    for tok in s.split():
        k, v = tok.split("=")
        out[k] = tuple(int(x) for x in v.split("x")) if "x" in v else int(v)
    return out


def kernel_of(plan):
    """('gemm', variant, width) or ('halo', kind, wide) of a parsed plan."""
    if plan["variant"] >= 0:
        return ("gemm", plan["variant"], plan["block_n"])
    return ("halo", plan["halo_kind"], plan["halo_wide"])
