"""ctypes binding of ``libb200sd.so`` (the C-ABI in ``include/b200sd.h``) + thin torch-tensor
wrappers.  PyTorch is plumbing here (device memory, streams); every compute call goes through
the C-ABI.  There is NO fallback: a missing library or a failing call raises."""
from __future__ import annotations

import ctypes as C
import os
import weakref

import torch

_HERE = os.path.dirname(os.path.abspath(__file__))
_LIB_PATH = os.path.join(_HERE, "libb200sd.so")
_lib = None


class B200SDError(RuntimeError):
    pass


class GemmArgs(C.Structure):
    _fields_ = [
        ("mode", C.c_int32), ("m", C.c_int32), ("n", C.c_int32), ("c0", C.c_int32), ("c1", C.c_int32),
        ("n_img", C.c_int32), ("h", C.c_int32), ("w", C.c_int32), ("stride", C.c_int32),
        ("geglu", C.c_int32), ("out_f32", C.c_int32), ("bias_rows", C.c_int32), ("bias_stride", C.c_int32),
        ("split_k", C.c_int32),
        ("block_n", C.c_int32), ("act", C.c_int32), ("wgt_tiled", C.c_int32), ("pad_after_only", C.c_int32),
        ("a0", C.c_void_p), ("a1", C.c_void_p), ("wgt", C.c_void_p), ("bias", C.c_void_p),
        ("residual", C.c_void_p), ("out", C.c_void_p), ("workspace", C.c_void_p),
        ("workspace_bytes", C.c_size_t),
        # fused normalisation (include/b200sd.h): halo convolution + GroupNorm operand transform, statistics outputs,
        # LayerNorm fold
        ("halo", C.c_int32), ("upsample2x", C.c_int32), ("gn_groups", C.c_int32), ("gn_silu", C.c_int32),
        ("gn_eps", C.c_float),
        ("gn_chan0", C.c_void_p), ("gn_chan1", C.c_void_p), ("gn_gamma", C.c_void_p), ("gn_beta", C.c_void_p),
        ("cs_partial", C.c_void_p), ("cs_chan", C.c_void_p), ("cs_tickets", C.c_void_p), ("cs_hw", C.c_int32),
        ("rs_out", C.c_void_p),
        ("ln_stat", C.c_void_p), ("ln_wg", C.c_void_p), ("ln_parts", C.c_int32), ("ln_eps", C.c_float),
        ("a2", C.c_void_p), ("a3", C.c_void_p), ("c2", C.c_int32), ("c3", C.c_int32),
        ("out_s8_inv_scale", C.c_float),  # > 0: int8 output (the operand of a W8A8 consumer)
    ]


class LutArgs(C.Structure):
    """b200sd_lut_args: the palettized B operand of b200sd_gemm_lut."""
    _fields_ = [("packed", C.c_void_p), ("lut", C.c_void_p), ("kscale", C.c_void_p), ("nbits", C.c_int32),
                ("row_bytes", C.c_int32), ("seg_end0", C.c_int32), ("seg_end1", C.c_int32)]


class StepCoeffs(C.Structure):
    _fields_ = [
        ("guidance", C.c_float), ("cx", C.c_float), ("ce", C.c_float), ("ch", C.c_float * 4),
        ("x0_cx", C.c_float), ("x0_ce", C.c_float), ("x0_ch", C.c_float * 4), ("n_hist", C.c_int32),
        ("push_eps_slot", C.c_int32), ("push_x0_slot", C.c_int32), ("push_x_slot", C.c_int32),
        ("noise_pred_nhwc", C.c_int32),
    ]


class BlendArgs(C.Structure):
    _fields_ = [("mask", C.c_void_p), ("image_latents", C.c_void_p), ("noise", C.c_void_p), ("a", C.c_float),
                ("b", C.c_float)]


_SIGNATURES = {
    "b200sd_last_error": (C.c_char_p, []),
    "b200sd_version": (C.c_int, []),
    "b200sd_launch_count": (C.c_uint64, []),
    "b200sd_set_pdl": (None, [C.c_int]),
    "b200sd_set_launch_classes": (None, [C.c_uint32]),
    # model-level handles (capi.py holds the struct mirrors)
    "b200sd_unet_create": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int32, C.c_void_p, C.c_void_p]),
    "b200sd_unet_prepare_prompt": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p]),
    "b200sd_unet_forward": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int32, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p,
                                      C.c_void_p, C.c_void_p, C.c_void_p]),
    "b200sd_unet_set_attention_impl": (C.c_int, [C.c_void_p, C.c_int32]),
    "b200sd_unet_device_bytes": (C.c_size_t, [C.c_void_p]),
    "b200sd_destroy": (None, [C.c_void_p]),
    "b200sd_gemm": (C.c_int, [C.POINTER(GemmArgs), C.c_void_p]),
    "b200sd_gemm_workspace_bytes": (C.c_size_t, [C.POINTER(GemmArgs)]),
    "b200sd_gemm_plan": (C.c_int, [C.POINTER(GemmArgs), C.POINTER(C.c_int32)]),
    "b200sd_gemm_plan_ex": (C.c_int, [C.POINTER(GemmArgs), C.POINTER(C.c_int32)]),
    "b200sd_gemm_describe_plan": (C.c_int, [C.POINTER(GemmArgs), C.c_char_p, C.c_size_t]),
    "b200sd_linear_small": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int32,
                                      C.c_int32, C.c_int32, C.c_int32, C.c_int32, C.c_void_p]),
    "b200sd_timestep_embedding": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int32, C.c_int32, C.c_int32, C.c_float,
                                            C.c_void_p]),
    "b200sd_group_norm": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int32, C.c_int32, C.c_int32, C.c_int32, C.c_int32,
                                    C.c_float, C.c_void_p, C.c_void_p, C.c_int32, C.c_void_p, C.c_void_p,
                                    C.c_size_t, C.c_void_p]),
    "b200sd_group_norm_workspace_bytes": (C.c_size_t, [C.c_int32, C.c_int32, C.c_int32, C.c_int32]),
    "b200sd_group_norm_apply": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int32, C.c_int32, C.c_int32, C.c_int32, C.c_int32,
                                          C.c_float, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int32, C.c_void_p,
                                          C.c_void_p]),
    "b200sd_layer_norm": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int32, C.c_int32,
                                    C.c_float, C.c_void_p]),
    "b200sd_softmax_rows": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int32, C.c_int32, C.c_float, C.c_void_p]),
    "b200sd_latent_prep": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_float, C.c_void_p, C.c_int32, C.c_int32,
                                     C.c_int32, C.c_int32, C.c_int32, C.c_void_p]),
    "b200sd_attention": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int32,
                                   C.c_int32, C.c_int32, C.c_int32, C.c_int32, C.c_int32, C.c_int32, C.c_int32,
                                   C.c_int32, C.c_float, C.c_int32, C.c_void_p]),
    "b200sd_attention_workspace_bytes": (C.c_size_t, []),
    "b200sd_attention_workspace_bytes_for": (C.c_size_t, [C.c_int32]),
    "b200sd_attention_ws": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int32,
                                      C.c_int32, C.c_int32, C.c_int32, C.c_int32, C.c_int32, C.c_int32, C.c_int32,
                                      C.c_int32, C.c_float, C.c_int32, C.c_void_p, C.c_size_t, C.c_void_p]),
    "b200sd_nchw_to_nhwc": (C.c_int, [C.c_void_p, C.c_int32, C.c_void_p, C.c_int32, C.c_int32, C.c_int32,
                                      C.c_int32, C.c_int32, C.c_void_p]),
    "b200sd_nhwc_to_nchw_f32": (C.c_int, [C.c_void_p, C.c_int32, C.c_void_p, C.c_int32, C.c_int32, C.c_int32,
                                          C.c_int32, C.c_int32, C.c_void_p]),
    "b200sd_upsample2x": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int32, C.c_int32, C.c_int32, C.c_int32,
                                    C.c_void_p]),
    "b200sd_add": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_size_t, C.c_void_p]),
    "b200sd_control_inject": (C.c_int, [C.c_void_p, C.POINTER(C.c_void_p), C.c_void_p, C.c_int32, C.c_void_p,
                                        C.c_size_t, C.c_void_p]),
    # W8A8 (int8 wgmma) 3x3 convolution and its operand producers
    "b200sd_gemm_s8": (C.c_int, [C.POINTER(GemmArgs), C.c_void_p, C.c_void_p]),
    "b200sd_gemm_lut": (C.c_int, [C.POINTER(GemmArgs), C.POINTER(LutArgs), C.c_void_p]),
    "b200sd_gemm_describe_plan_lut": (C.c_int, [C.POINTER(GemmArgs), C.POINTER(LutArgs), C.c_char_p, C.c_size_t]),
    "b200sd_gemm_plan_ex_s8": (C.c_int, [C.POINTER(GemmArgs), C.POINTER(C.c_int32)]),
    "b200sd_gemm_describe_plan_s8": (C.c_int, [C.POINTER(GemmArgs), C.c_char_p, C.c_size_t]),
    "b200sd_gemm_workspace_bytes_s8": (C.c_size_t, [C.POINTER(GemmArgs)]),
    "b200sd_gemm_s8_linear": (C.c_int, [C.POINTER(GemmArgs), C.c_void_p, C.c_void_p]),
    "b200sd_gemm_plan_ex_s8_linear": (C.c_int, [C.POINTER(GemmArgs), C.POINTER(C.c_int32)]),
    "b200sd_gemm_describe_plan_s8_linear": (C.c_int, [C.POINTER(GemmArgs), C.c_char_p, C.c_size_t]),
    "b200sd_gemm_workspace_bytes_s8_linear": (C.c_size_t, [C.POINTER(GemmArgs)]),
    "b200sd_layer_norm_s8": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_float, C.c_void_p, C.c_int32, C.c_int32,
                                       C.c_float, C.c_void_p]),
    "b200sd_group_norm_s8": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int32, C.c_int32, C.c_int32, C.c_int32, C.c_int32,
                                       C.c_float, C.c_void_p, C.c_void_p, C.c_int32, C.c_float, C.c_void_p, C.c_void_p,
                                       C.c_size_t, C.c_void_p]),
    "b200sd_upsample2x_s8": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int32, C.c_int32, C.c_int32, C.c_int32, C.c_float,
                                       C.c_void_p]),
    "b200sd_absmax_f16": (C.c_int, [C.c_void_p, C.c_size_t, C.c_void_p, C.c_void_p]),
    "b200sd_ctx_to_tokens": (C.c_int, [C.c_void_p, C.c_int32, C.c_void_p, C.c_int32, C.c_int32, C.c_int32,
                                       C.c_void_p]),
    "b200sd_embed_tokens": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int32, C.c_int32, C.c_int32,
                                      C.c_int32, C.c_void_p]),
    "b200sd_cfg_scheduler_step": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int32,
                                            C.c_int32, C.c_int32, C.c_int32, C.c_int32, C.POINTER(StepCoeffs),
                                            C.c_void_p]),
    "b200sd_cfg_scheduler_step_noised": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p,
                                                   C.c_int32, C.c_int32, C.c_int32, C.c_int32, C.c_int32,
                                                   C.POINTER(StepCoeffs), C.c_float, C.c_void_p, C.c_uint32,
                                                   C.c_void_p]),
    "b200sd_cfg_scheduler_step_blend": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p,
                                                  C.c_int32, C.c_int32, C.c_int32, C.c_int32, C.c_int32,
                                                  C.POINTER(StepCoeffs), C.c_float, C.c_void_p, C.c_uint32,
                                                  C.POINTER(BlendArgs), C.c_void_p]),
    "b200sd_scheduler_step_guidance_free": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p,
                                                      C.c_int32, C.c_int32, C.c_int32, C.c_int32, C.c_int32,
                                                      C.POINTER(StepCoeffs), C.c_float, C.c_void_p, C.c_uint32,
                                                      C.POINTER(BlendArgs), C.c_void_p]),
    "b200sd_image_postprocess":(C.c_int, [C.c_void_p, C.c_int32, C.c_int32, C.c_void_p, C.c_void_p, C.c_int32,
                                           C.c_int32, C.c_int32, C.c_int32, C.c_void_p]),
    # safety checker (csrc/vision.cu)
    "b200sd_clip_preprocess": (C.c_int, [C.c_void_p, C.c_int32, C.c_int32, C.c_int32, C.c_void_p, C.c_void_p,
                                         C.c_void_p, C.c_int32, C.c_void_p, C.c_void_p, C.c_int32, C.c_int32,
                                         C.c_int32, C.POINTER(C.c_float), C.POINTER(C.c_float), C.c_void_p,
                                         C.c_void_p]),
    "b200sd_patchify": (C.c_int, [C.c_void_p, C.c_int32, C.c_int32, C.c_int32, C.c_int32, C.c_int32, C.c_void_p,
                                  C.c_void_p]),
    "b200sd_safety_concepts": (C.c_int, [C.c_void_p, C.c_int32, C.c_int32, C.c_void_p, C.c_void_p, C.c_int32,
                                         C.c_void_p, C.c_void_p, C.c_int32, C.c_void_p, C.c_void_p, C.c_void_p,
                                         C.c_void_p]),
    "b200sd_filter_images": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int32, C.c_int32, C.c_int32,
                                       C.c_int32, C.c_void_p]),
}
# bf16 twins (include/b200sd.h): same signatures, every fp16 pointer is bf16
for _name in ("b200sd_gemm", "b200sd_gemm_plan_ex", "b200sd_gemm_describe_plan", "b200sd_group_norm",
              "b200sd_softmax_rows", "b200sd_latent_prep", "b200sd_nchw_to_nhwc"):
    _SIGNATURES[_name + "_bf16"] = _SIGNATURES[_name]
del _name

EXPORTED_SYMBOLS = tuple(_SIGNATURES)


def lib_path() -> str:
    return _LIB_PATH


def load():
    """Load the CUDA library; raise loudly if it has not been built (no CPU fallback exists)."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(_LIB_PATH):
        raise B200SDError(
            f"{_LIB_PATH} is missing: build it with `python -c 'import __graft_entry__ as g; g.build()'` "
            "(nvcc, sm_90a). b200sd has no CPU or PyTorch fallback path.")
    lib = C.CDLL(_LIB_PATH)
    for name, (res, args) in _SIGNATURES.items():
        fn = getattr(lib, name)  # AttributeError if the symbol is not exported
        fn.restype = res
        fn.argtypes = args
    _lib = lib
    return lib


def _stream():
    return C.c_void_p(torch.cuda.current_stream().cuda_stream)


def _ptr(t):
    if t is None:
        return None
    return C.c_void_p(t.data_ptr())


_DEBUG_SYNC = bool(os.environ.get("B200SD_DEBUG_SYNC"))


def _check(rc, what):
    if rc != 0:
        msg = load().b200sd_last_error().decode(errors="replace")
        raise B200SDError(f"{what} failed (rc={rc}): {msg}")
    if _DEBUG_SYNC:  # debugging aid: localise a faulting / hanging kernel
        print(f"[b200sd] {what} launched", flush=True)
        torch.cuda.synchronize()
        print(f"[b200sd] {what} done", flush=True)


def launch_count() -> int:
    return int(load().b200sd_launch_count())


# ------------------------------------------------------------------------------------------------
# op wrappers (torch tensors in, torch tensors out; all on the current CUDA stream)
# ------------------------------------------------------------------------------------------------
def _req(t, dtype, what):
    if t.dtype != dtype or not t.is_cuda or not t.is_contiguous():
        raise B200SDError(f"{what}: expected contiguous CUDA {dtype}, got {t.dtype} {t.device} "
                          f"contiguous={t.is_contiguous()}")


ACT_DTYPES = (torch.float16, torch.bfloat16)  # bf16: the VAEs whose activations overflow fp16 (force_upcast)


def _act_dtype(x, what):
    """The 16-bit type a call runs in: its input's (bf16, else fp16, which _req then demands)."""
    dt = torch.bfloat16 if x.dtype == torch.bfloat16 else torch.float16
    _req(x, dt, what)
    return dt


def _same16(dt, a, b, what):
    """Every 16-bit operand of one call shares the input's type (a, b: optional operands)."""
    if (a is not None and a.dtype != dt) or (b is not None and b.dtype != dt):
        raise B200SDError(f"{what}: operand types differ in a {dt} call (all 16-bit operands share one type)")


def _sfx(dt):
    return "_bf16" if dt == torch.bfloat16 else ""


def gemm_args(mode, a0, wgt, out, *, a1=None, bias=None, residual=None, m=0, n=0, n_img=0, h=0, w=0, stride=1,
              geglu=False, bias_rows=0, bias_stride=0, split_k=0, block_n=0, workspace=None, act=0, pad_after_only=False):
    args = GemmArgs()
    args.mode = mode
    args.m = m
    args.n = n
    args.c0 = a0.shape[-1]
    args.c1 = 0 if a1 is None else a1.shape[-1]
    args.n_img, args.h, args.w, args.stride = n_img, h, w, stride
    args.geglu = int(geglu)
    args.out_f32 = int(out.dtype == torch.float32)
    args.bias_rows = bias_rows
    args.bias_stride = bias_stride
    args.split_k = split_k
    args.block_n = block_n
    args.act = act
    args.pad_after_only = int(pad_after_only)
    args.a0 = a0.data_ptr()
    args.a1 = None if a1 is None else a1.data_ptr()
    args.wgt = wgt.data_ptr()
    args.bias = None if bias is None else bias.data_ptr()
    args.residual = None if residual is None else residual.data_ptr()
    args.out = out.data_ptr()
    args.workspace = None if workspace is None else workspace.data_ptr()
    args.workspace_bytes = 0 if workspace is None else workspace.numel() * workspace.element_size()
    return args


def describe_plan(mode, m=0, n=0, c0=0, c1=0, n_img=0, h=0, w=0, stride=1, geglu=False, has_bias=True,
                  has_residual=False, bias_rows=0, split_k=0, block_n=0, out_f32=False, act=0, pad_after_only=False,
                  rowstats=False, stats=False, cs_hw=0, ln=False, c2=0, c3=0, halo=0, upsample=False, gn=False,
                  bf16=False, out_s8=False) -> str:
    """Host-only: the tiling the launcher would choose (no GPU needed).  The flags mirror linear() / conv3x3():
    rowstats / stats (with cs_hw, the rows per image of a linear) ask for the statistics outputs, ln for the LayerNorm
    fold, c2 / c3 are the folded shortcut's channels, halo / upsample / gn select the halo convolution (mode 0 with halo:
    its 1x1 form; m = n_img * h * w); bf16 plans the bf16 call (b200sd_gemm_bf16); out_s8 an int8 output."""
    a = GemmArgs()
    a.mode, a.m, a.n, a.c0, a.c1, a.n_img, a.h, a.w, a.stride = mode, m, n, c0, c1, n_img, h, w, stride
    a.geglu, a.bias_rows, a.split_k, a.block_n = int(geglu), bias_rows, split_k, block_n
    a.out_f32, a.act, a.pad_after_only = int(out_f32), act, int(pad_after_only)
    # pointers are only tested for null-ness by the planner
    a.bias = 1 if has_bias else None
    a.residual = 1 if has_residual else None
    if stats:
        a.cs_partial, a.cs_hw = 1, cs_hw
    if rowstats:
        a.rs_out = 1
    if ln:
        a.ln_stat, a.ln_wg, a.ln_parts = 1, 1, 1
    a.c2, a.c3 = c2, c3
    a.halo, a.upsample2x, a.gn_groups = int(halo), int(upsample), 32 if gn else 0
    a.out_s8_inv_scale = 1.0 if out_s8 else 0.0
    if stats or rowstats or ln or gn:
        a.split_k = 1  # as linear() / conv3x3() ask for the fused outputs
    buf = C.create_string_buffer(512)
    name = "b200sd_gemm_describe_plan" + ("_bf16" if bf16 else "")
    _check(getattr(load(), name)(C.byref(a), buf, 512), name)
    return buf.value.decode()


TILED_WEIGHTS = os.environ.get("B200SD_TILED_W", "1") != "0"
_tiled_cache = {}  # key -> (weakref to the source weight, its _version, packed copy)


def _cache_tiled(key, wgt, packed):
    """Cache `packed` for as long as its source tensor lives: the entry (and the packed device copy) is dropped when
    `wgt` is freed, so the tiled weights of a model that is gone do not stay resident.  A lookup only ever hits the
    live source tensor itself, so nothing is lost."""
    def drop(ref, key=key):
        if _tiled_cache.get(key, (None,))[0] is ref:  # not an entry a newer tensor at the same address has taken
            del _tiled_cache[key]

    _tiled_cache[key] = (weakref.ref(wgt, drop), wgt._version, packed)


def pack_tiled(w2d, c0, c1, taps, bn, chunk_major=False, extra=(0, 0), chunk=64):
    """[N, taps*(c0+c1) (+ c2 + c3)] -> [n_tiles, k_blocks, bn, 64] fp16 in the exact k-block order of the kernel's main
    loop (tap-major; per tap the 64-channel chunks of source 0, then of source 1; ragged chunks zero padded), so
    that each weight tile is one contiguous bn*128-byte burst in HBM.  chunk_major: k-block = chunk * taps + tap
    (the halo convolution walks all nine taps of one 64-channel chunk before the next chunk).  extra = (c2, c3): the
    folded shortcut's columns follow the convolution's: their chunks (source 2, then source 3) are the last k-blocks.
    chunk: channels per k-block (128 for the int8 convolution, whose k-block is the same 128 bytes)."""
    n, kpt = w2d.shape[0], c0 + c1
    kc0, kc1 = (c0 + chunk - 1) // chunk, (c1 + chunk - 1) // chunk
    kc = kc0 + kc1
    nt = (n + bn - 1) // bn
    c2, c3 = extra
    wp = torch.zeros(nt * bn, taps, kpt, dtype=w2d.dtype, device=w2d.device)
    wp[:n] = w2d[:, : taps * kpt].reshape(n, taps, kpt)
    out = torch.zeros(nt, taps, kc, bn, chunk, dtype=w2d.dtype, device=w2d.device)
    for j in range(kc):
        lo = j * chunk if j < kc0 else c0 + (j - kc0) * chunk
        hi = min(lo + chunk, c0 if j < kc0 else kpt)
        out[:, :, j, :, : hi - lo] = wp[:, :, lo:hi].reshape(nt, bn, taps, hi - lo).permute(0, 2, 1, 3)
    if chunk_major:
        out = out.permute(0, 2, 1, 3, 4)
    out = out.reshape(nt, taps * kc, bn, chunk)
    if c2 + c3:
        if chunk_major:
            raise B200SDError("pack_tiled: shortcut columns are not supported in the chunk-major (halo) layout")
        kc2, kc3 = (c2 + 63) // 64, (c3 + 63) // 64
        we = torch.zeros(nt * bn, c2 + c3, dtype=w2d.dtype, device=w2d.device)
        we[:n] = w2d[:, taps * kpt:]
        ext = torch.zeros(nt, kc2 + kc3, bn, 64, dtype=w2d.dtype, device=w2d.device)
        for j in range(kc2 + kc3):
            lo = j * 64 if j < kc2 else c2 + (j - kc2) * 64
            hi = min(lo + 64, c2 if j < kc2 else c2 + c3)
            ext[:, j, :, : hi - lo] = we[:, lo:hi].reshape(nt, bn, hi - lo)
        out = torch.cat([out, ext], 1)
    return out.contiguous()


def plan_ex(args, bf16=False):
    """(block_n, splits, kb_total, n_tiles, stat slots per image, staged, stages, m_tiles) of a call."""
    plan = (C.c_int32 * 8)()
    name = "b200sd_gemm_plan_ex" + ("_bf16" if bf16 else "")
    _check(getattr(load(), name)(C.byref(args), plan), name)
    return tuple(int(v) for v in plan)


def _maybe_tile_weights(args, wgt, taps):
    """Static weight operands are re-laid out once per (weight, block_n) and cached."""
    bn = plan_ex(args, bf16=wgt.dtype == torch.bfloat16)[0]
    key = (wgt.data_ptr(), bn, args.c0, args.c1, taps, bool(args.halo), args.c2, args.c3)
    hit = _tiled_cache.get(key)
    packed = None
    if hit is not None and hit[0]() is wgt and hit[1] == wgt._version:
        packed = hit[2]
    if packed is None:
        if torch.cuda.is_current_stream_capturing():
            return  # never pack during capture; the warm-up pass has populated the cache for these shapes
        packed = pack_tiled(wgt, args.c0, args.c1, taps, bn, chunk_major=bool(args.halo), extra=(args.c2, args.c3))
        _cache_tiled(key, wgt, packed)
    args.wgt = packed.data_ptr()
    args.block_n = bn
    args.wgt_tiled = 1


def lut_args(pw):
    """LutArgs of a palettization.PalettizedWeight."""
    la = LutArgs()
    la.packed, la.lut = pw.packed.data_ptr(), pw.lut.data_ptr()
    la.kscale = None if pw.kscale is None else pw.kscale.data_ptr()
    la.nbits, la.row_bytes = pw.nbits, pw.packed.shape[1]
    la.seg_end0, la.seg_end1 = pw.seg_ends
    return la


def describe_plan_lut(args, pw) -> str:
    """Host-only: the tiling b200sd_gemm_lut would choose for these args and palettized weight."""
    buf = C.create_string_buffer(512)
    _check(load().b200sd_gemm_describe_plan_lut(C.byref(args), C.byref(lut_args(pw)), buf, 512),
           "b200sd_gemm_describe_plan_lut")
    return buf.value.decode()


def _is_lut(wgt):
    return hasattr(wgt, "packed") and hasattr(wgt, "lut")


def _run_gemm_lut(args, pw, device):
    """b200sd_gemm_lut: `pw` (a palettization.PalettizedWeight) is the B operand, on the fp16 plan of `args`."""
    args.wgt, args.wgt_tiled = None, 0
    need = gemm_workspace_bytes(args)
    if need:
        ws = _workspace(need, device)
        args.workspace = ws.data_ptr()
        args.workspace_bytes = ws.numel() * 4
    _check(load().b200sd_gemm_lut(C.byref(args), C.byref(lut_args(pw)), _stream()), "b200sd_gemm_lut")


def gemm_workspace_bytes(args) -> int:
    return int(load().b200sd_gemm_workspace_bytes(C.byref(args)))


def run_gemm(args):
    _check(load().b200sd_gemm(C.byref(args), _stream()), "b200sd_gemm")


def run_gemm_bf16(args):
    _check(load().b200sd_gemm_bf16(C.byref(args), _stream()), "b200sd_gemm_bf16")


def _check_out(out, dt, what):
    if out is not None and out.dtype not in (dt, torch.float32):
        raise B200SDError(f"{what}: {out.dtype} output in a {dt} call (fp32 or the input's type)")


_ws_cache = {}
_ws_retired = []   # superseded workspaces stay allocated: CUDA graphs captured earlier hold their addresses
_ticket_cache = {}


def _workspace(nbytes, device):
    """Process-wide scratch (split-K partials, GroupNorm / column-statistics partials).  Kernels that use it are
    stream-ordered on the single compute stream of the process.  It only ever grows (outside of CUDA-graph
    capture: the warm-up pass sizes it) and a superseded buffer is never freed, so pointers baked into
    previously captured graphs stay valid."""
    key = device.index
    ws = _ws_cache.get(key)
    if ws is None or ws.numel() * 4 < nbytes:
        if torch.cuda.is_current_stream_capturing():
            raise B200SDError("workspace would have to grow during CUDA-graph capture; run one eager "
                              "warm-up call with the same shapes first")
        if ws is not None:
            _ws_retired.append(ws)
        ws = torch.empty(max(nbytes // 4 + 1, 1 << 24), dtype=torch.float32, device=device)
        _ws_cache[key] = ws
    return ws


def _tickets(device):
    """Arrival counters of the statistics epilogue ([n_img][n_tiles] per call): zero once, self-resetting, shared by
    every call on the device (calls are stream ordered)."""
    t = _ticket_cache.get(device.index)
    if t is None:
        t = torch.zeros(1 << 16, dtype=torch.int32, device=device)
        _ticket_cache[device.index] = t
    return t


def _fused_args(args, x_dev, *, n_img, cout, gn=None, stats=None, cs_hw=0, ln=None, rowstats=None, m=0):
    """Fill the fused-normalisation fields of a GemmArgs.  gn: dict(chan0, chan1, gamma, beta, groups, eps, silu);
    stats: dict, receives 'chan' [n_img, cout, 2]; rowstats: dict, receives 'rows' [n_tiles, m, 2] and 'parts';
    ln: dict(stat, parts, wg, eps)."""
    keep = []
    if gn is not None:
        args.gn_groups, args.gn_silu, args.gn_eps = int(gn["groups"]), int(bool(gn["silu"])), float(gn["eps"])
        args.gn_chan0 = gn["chan0"].data_ptr()
        args.gn_chan1 = None if gn.get("chan1") is None else gn["chan1"].data_ptr()
        args.gn_gamma, args.gn_beta = gn["gamma"].data_ptr(), gn["beta"].data_ptr()
    if ln is not None:
        args.ln_stat, args.ln_wg = ln["stat"].data_ptr(), ln["wg"].data_ptr()
        args.ln_parts, args.ln_eps = int(ln["parts"]), float(ln.get("eps", 1e-5))
    if stats is not None or rowstats is not None:
        if stats is not None:
            args.cs_partial = 1  # planning query: non-null
            args.cs_hw = cs_hw
        if rowstats is not None:
            args.rs_out = 1
        try:
            pl = plan_ex(args)
        except B200SDError:
            if stats is None:
                raise
            # this geometry cannot emit column statistics (e.g. images smaller than 16 pixels): the caller sees no
            # 'chan' entry and its consumer falls back to the standalone GroupNorm kernel
            args.cs_partial, args.cs_hw, stats = None, 0, None
            if rowstats is None:
                return keep
            pl = plan_ex(args)
        n_tiles, slots = pl[3], pl[4]
        if stats is not None:
            if n_img * n_tiles > (1 << 16):
                raise B200SDError("statistics ticket table too small")
            chan = torch.empty(n_img, cout, 2, dtype=torch.float32, device=x_dev)
            part = _workspace(n_img * slots * cout * 2 * 4, x_dev)
            args.cs_partial, args.cs_chan, args.cs_tickets = part.data_ptr(), chan.data_ptr(), _tickets(x_dev).data_ptr()
            stats["chan"] = chan
            keep.append(chan)
        if rowstats is not None:
            parts = n_tiles if pl[5] else 2 * n_tiles  # register epilogue: one partial per column half of a tile
            rows = torch.empty(parts, m, 2, dtype=torch.float32, device=x_dev)
            args.rs_out = rows.data_ptr()
            rowstats["rows"], rowstats["parts"] = rows, parts
            keep.append(rows)
    return keep


def linear(x, wgt, bias=None, residual=None, *, x1=None, geglu=False, out_dtype=None, split_k=0,
           block_n=0, bias_rows=0, bias_stride=0, out=None, static_w=False, act=0, ln=None, stats=None, cs_hw=0,
           rowstats=None, out_inv_scale=None):
    """out[M, N] = epilogue([x | x1] @ wgt^T).  x [M, C0] fp16, wgt [N, C0(+C1)] fp16, bias fp32 [N].
    x bf16 runs the bf16 kernels: then wgt, x1, residual and a 16-bit output are bf16 too (out_dtype None: x's type).
    static_w: `wgt` is a model weight (constant address/content) and may be re-tiled + cached.
    ln: LayerNorm of x folded into this GEMM (wgt = gamma (.) W, bias = W beta + b; dict(stat, parts, wg, eps));
    stats / rowstats: dicts that receive the per-channel / per-row sums of the output (see _fused_args).
    out_inv_scale: int8 output q = clamp(rint(y * out_inv_scale), -127, 127) for a W8A8 consumer (fp16 x)."""
    dt = _act_dtype(x, "linear x")
    lut = _is_lut(wgt)
    if lut:
        if dt != torch.float16:
            raise B200SDError("linear: palettized weights need fp16 activations")
    else:
        _req(wgt, dt, "linear wgt")
    _same16(dt, x1, residual, "linear x1 / residual")
    m, n = x.shape[0], wgt.shape[0]
    n_out = n // 2 if geglu else n
    if out_inv_scale is not None:
        out_dtype = torch.int8
    if out is None:
        out = torch.empty(m, n_out, dtype=out_dtype or dt, device=x.device)
    if out_inv_scale is None:
        _check_out(out, dt, "linear out")
    else:
        _req(out, torch.int8, "linear out (int8 output)")
    args = gemm_args(0, x, wgt.packed if lut else wgt, out, a1=x1, bias=bias, residual=residual, m=m, n=n, geglu=geglu,
                     bias_rows=bias_rows, bias_stride=bias_stride, split_k=split_k, block_n=block_n, act=act)
    if out_inv_scale is not None:
        args.out_s8_inv_scale = float(out_inv_scale)
    if ln is not None or stats is not None or rowstats is not None:
        args.split_k = 1
        _keep = _fused_args(args, x.device, n_img=(m // cs_hw if cs_hw else 0), cout=n, stats=stats, cs_hw=cs_hw, ln=ln,
                            rowstats=rowstats, m=m)
    if lut:
        _run_gemm_lut(args, wgt, x.device)
        return out
    if static_w and TILED_WEIGHTS:
        _maybe_tile_weights(args, wgt, 1)
    bf16 = dt == torch.bfloat16
    need = 0 if bf16 else gemm_workspace_bytes(args)  # bf16 never splits K
    if need:
        ws = _workspace(need, x.device)
        args.workspace = ws.data_ptr()
        args.workspace_bytes = ws.numel() * 4
    if bf16:
        run_gemm_bf16(args)
    else:
        run_gemm(args)
    return out


def conv3x3(x, wgt, bias=None, residual=None, *, x1=None, stride=1, out_dtype=None, split_k=0,
            block_n=0, bias_rows=0, bias_stride=0, out=None, act=0, static_w=True, pad_after_only=False,
            halo=False, gn=None, upsample=False, stats=None, rowstats=None, taps=9, shortcut=None):
    """3x3 pad-1 convolution.  x NHWC fp16 [N, H, W, C0]; wgt [Cout, 9*(C0+C1)] fp16 (OHWI);
    bias fp32 [Cout] or [N_img, Cout] with bias_rows = Hout*Wout.
    halo: the halo-reuse kernel (stride 1); gn: GroupNorm (+SiLU) of x ++ x1 applied while loading (dict(chan0, chan1,
    gamma, beta, groups, eps, silu), needs halo); upsample: x is read nearest-x2 upsampled (halo); stats: dict that
    receives 'chan', the per-channel (sum, sum of squares) of the output for the consumer's GroupNorm; taps=1 with
    halo: a 1x1 convolution (wgt [Cout, C0+C1]) that shares the halo kernel's GroupNorm operand path.
    shortcut = (s0, s1 or None): the ResNet shortcut folded in -- wgt is [Cout, 9*(C0+C1) + Cs0 + Cs1] (the 1x1
    shortcut matrix appended along K), bias the sum of both biases, s0 / s1 NHWC fp16 at the output resolution.
    x bf16 runs the bf16 kernels (no halo / gn / upsample / stats / shortcut): wgt, x1, residual and a 16-bit output
    are bf16 too (out_dtype None: x's type)."""
    dt = _act_dtype(x, "conv3x3 x")
    lut = _is_lut(wgt)
    if lut:
        if dt != torch.float16 or halo or shortcut is not None:
            raise B200SDError("conv3x3: palettized weights need fp16 activations and the 9-tap kernel without a folded shortcut")
    else:
        _req(wgt, dt, "conv3x3 wgt")
    _same16(dt, x1, residual, "conv3x3 x1 / residual")
    nimg, h, w, _ = x.shape
    if upsample:
        h, w = 2 * h, 2 * w
    cout = wgt.shape[0]
    ho, wo = h // stride, w // stride
    if out is None:
        out = torch.empty(nimg, ho, wo, cout, dtype=out_dtype or dt, device=x.device)
    _check_out(out, dt, "conv3x3 out")
    if (gn is not None or upsample or taps == 1) and not halo:
        raise B200SDError("conv3x3: gn / upsample / taps=1 need halo=True")
    args = gemm_args(1 if taps == 9 else 0, x, wgt.packed if lut else wgt, out, a1=x1, bias=bias, residual=residual, n=cout, n_img=nimg, h=h, w=w,
                     stride=stride, bias_rows=bias_rows, bias_stride=bias_stride, split_k=split_k, block_n=block_n, act=act,
                     pad_after_only=pad_after_only, m=(nimg * h * w if taps == 1 else 0))
    args.halo, args.upsample2x = int(halo), int(upsample)
    if shortcut is not None:
        s0, s1 = shortcut
        if stride != 1 or taps != 9 or halo or not (static_w and TILED_WEIGHTS):
            raise B200SDError("conv3x3: a folded shortcut needs the stride-1 9-tap kernel with static pre-tiled weights")
        _req(s0, dt, "conv3x3 shortcut source")
        args.a2, args.c2 = s0.data_ptr(), s0.shape[-1]
        if s1 is not None:
            _req(s1, dt, "conv3x3 shortcut source 1")
            args.a3, args.c3 = s1.data_ptr(), s1.shape[-1]
    _keep = None
    if gn is not None or stats is not None or rowstats is not None:
        args.split_k = 1
        _keep = _fused_args(args, x.device, n_img=nimg, cout=cout, gn=gn, stats=stats, cs_hw=ho * wo, rowstats=rowstats,
                            m=nimg * ho * wo)
    if lut:
        _run_gemm_lut(args, wgt, x.device)
        return out
    if halo and not (static_w and TILED_WEIGHTS):
        raise B200SDError("conv3x3: the halo kernel needs static pre-tiled weights")
    if static_w and TILED_WEIGHTS:
        _maybe_tile_weights(args, wgt, taps)
    bf16 = dt == torch.bfloat16
    need = 0 if bf16 else gemm_workspace_bytes(args)  # bf16 never splits K
    if need:
        ws = _workspace(need, x.device)
        args.workspace = ws.data_ptr()
        args.workspace_bytes = ws.numel() * 4
    if bf16:
        run_gemm_bf16(args)
    else:
        run_gemm(args)
    return out


# ------------------------------------------------------------------------------------------------
# W8A8: int8 3x3 convolution (b200sd_gemm_s8) and the kernels that produce its int8 operand
# ------------------------------------------------------------------------------------------------
def plan_ex_s8(args):
    """plan_ex of the int8 convolution (k-blocks of 128 channels)."""
    plan = (C.c_int32 * 8)()
    _check(load().b200sd_gemm_plan_ex_s8(C.byref(args), plan), "b200sd_gemm_plan_ex_s8")
    return tuple(int(v) for v in plan)


def describe_plan_s8(n, c0, n_img, h, w, has_bias=True, has_residual=False, bias_rows=0, split_k=0, block_n=0) -> str:
    """Host-only: the tiling b200sd_gemm_s8 would choose for a stride-1 3x3 convolution (see describe_plan)."""
    a = GemmArgs()
    a.mode, a.n, a.c0, a.n_img, a.h, a.w, a.stride = 1, n, c0, n_img, h, w, 1
    a.bias_rows, a.split_k, a.block_n = bias_rows, split_k, block_n
    a.bias = 1 if has_bias else None
    a.residual = 1 if has_residual else None
    buf = C.create_string_buffer(512)
    _check(load().b200sd_gemm_describe_plan_s8(C.byref(a), buf, 512), "b200sd_gemm_describe_plan_s8")
    return buf.value.decode()


def _tiled_s8(args, wgt, taps=9):
    """int8 [Cout, taps*C0] (OHWI for the convolution) weights -> the pre-tiled layout of the planned width (cached per
    (weight, block_n))."""
    what = "conv3x3_s8" if taps == 9 else "linear_s8"
    bn = args.block_n if args.block_n > 0 else (plan_ex_s8 if taps == 9 else plan_ex_s8_linear)(args)[0]
    key = (wgt.data_ptr(), bn, args.c0, "s8") if taps == 9 else (wgt.data_ptr(), bn, args.c0, "s8_linear")
    hit = _tiled_cache.get(key)
    if hit is not None and hit[0]() is wgt and hit[1] == wgt._version:
        return hit[2], bn
    if torch.cuda.is_current_stream_capturing():
        raise B200SDError(f"{what}: weights of this shape were not tiled before CUDA-graph capture; run one eager "
                          "call with the same shapes first")
    packed = pack_tiled(wgt, args.c0, 0, taps, bn, chunk=128)
    _cache_tiled(key, wgt, packed)
    return packed, bn


def conv3x3_s8(x, wgt, col_scale, bias=None, residual=None, *, bias_rows=0, bias_stride=0, split_k=0, block_n=0,
               out=None):
    """W8A8 3x3 pad-1 stride-1 convolution on int8 wgmma.  x int8 NHWC [N, H, W, C] (C a multiple of 16); wgt int8
    [Cout, 9*C] (OHWI, symmetric per-output-channel quantized); col_scale fp32 [Cout] = s_a * s_w; bias fp32 [Cout] or
    [N, Cout] rows (bias_rows = H*W); residual fp16 NHWC [N, H, W, Cout].  Returns fp16 NHWC
    fp16(acc * col_scale + bias + residual)."""
    _req(x, torch.int8, "conv3x3_s8 x")
    _req(wgt, torch.int8, "conv3x3_s8 wgt")
    _req(col_scale, torch.float32, "conv3x3_s8 col_scale")
    if residual is not None:
        _req(residual, torch.float16, "conv3x3_s8 residual")
    nimg, h, w, c = x.shape
    cout = wgt.shape[0]
    if wgt.shape[1] != 9 * c or col_scale.numel() != cout:
        raise B200SDError(f"conv3x3_s8: weight {tuple(wgt.shape)} / col_scale {col_scale.numel()} do not match "
                          f"{c} input and {cout} output channels")
    if out is None:
        out = torch.empty(nimg, h, w, cout, dtype=torch.float16, device=x.device)
    _req(out, torch.float16, "conv3x3_s8 out")
    args = gemm_args(1, x, wgt, out, bias=bias, residual=residual, n=cout, n_img=nimg, h=h, w=w, bias_rows=bias_rows,
                     bias_stride=bias_stride, split_k=split_k, block_n=block_n)
    packed, bn = _tiled_s8(args, wgt)
    args.wgt, args.block_n, args.wgt_tiled = packed.data_ptr(), bn, 1
    need = int(load().b200sd_gemm_workspace_bytes_s8(C.byref(args)))
    if need:
        ws = _workspace(need, x.device)
        args.workspace = ws.data_ptr()
        args.workspace_bytes = ws.numel() * 4
    _check(load().b200sd_gemm_s8(C.byref(args), _ptr(col_scale), _stream()), "b200sd_gemm_s8")
    return out


def plan_ex_s8_linear(args):
    """plan_ex of the int8 linear GEMM (k-blocks of 128 channels)."""
    plan = (C.c_int32 * 8)()
    _check(load().b200sd_gemm_plan_ex_s8_linear(C.byref(args), plan), "b200sd_gemm_plan_ex_s8_linear")
    return tuple(int(v) for v in plan)


def describe_plan_s8_linear(m, n, c0, geglu=False, has_bias=True, has_residual=False, rowstats=False, out_s8=False,
                            split_k=0, block_n=0) -> str:
    """Host-only: the tiling b200sd_gemm_s8_linear would choose (see describe_plan); out_s8: int8 output."""
    a = GemmArgs()
    a.mode, a.m, a.n, a.c0, a.geglu, a.split_k, a.block_n = 0, m, n, c0, int(geglu), split_k, block_n
    a.bias = 1 if has_bias else None
    a.residual = 1 if has_residual else None
    if rowstats:
        a.rs_out, a.split_k = 1, 1
    if out_s8:
        a.out_s8_inv_scale = 1.0
    buf = C.create_string_buffer(512)
    _check(load().b200sd_gemm_describe_plan_s8_linear(C.byref(a), buf, 512), "b200sd_gemm_describe_plan_s8_linear")
    return buf.value.decode()


def linear_s8(x, wgt, col_scale, bias=None, residual=None, *, geglu=False, rowstats=None, out_inv_scale=None,
              split_k=0, block_n=0, out=None):
    """W8A8 linear on int8 wgmma.  x int8 [M, C] (C a multiple of 16); wgt int8 [N, C] (symmetric per-output-channel
    quantized; GEGLU: value / gate rows interleaved as for linear()); col_scale fp32 [N] = s_a * s_w; bias fp32 [N];
    residual fp16 [M, N_out].  y = acc * col_scale + bias (-> GEGLU) + residual, stored fp16, or int8
    clamp(rint(y * out_inv_scale), -127, 127) when out_inv_scale is given.  rowstats: dict that receives the per-row
    sums of the fp16 output for a LayerNorm folded into the consumer (see _fused_args)."""
    _req(x, torch.int8, "linear_s8 x")
    _req(wgt, torch.int8, "linear_s8 wgt")
    _req(col_scale, torch.float32, "linear_s8 col_scale")
    if residual is not None:
        _req(residual, torch.float16, "linear_s8 residual")
    m, c = x.shape
    n = wgt.shape[0]
    if wgt.shape[1] != c or col_scale.numel() != n:
        raise B200SDError(f"linear_s8: weight {tuple(wgt.shape)} / col_scale {col_scale.numel()} do not match {c} input "
                          f"and {n} output channels")
    out_dtype = torch.int8 if out_inv_scale is not None else torch.float16
    if out is None:
        out = torch.empty(m, n // 2 if geglu else n, dtype=out_dtype, device=x.device)
    _req(out, out_dtype, "linear_s8 out")
    args = gemm_args(0, x, wgt, out, bias=bias, residual=residual, m=m, n=n, geglu=geglu, split_k=split_k,
                     block_n=block_n)
    if out_inv_scale is not None:
        args.out_s8_inv_scale = float(out_inv_scale)
    _keep = None
    if rowstats is not None:
        args.rs_out, args.split_k = 1, 1
        pl = plan_ex_s8_linear(args)
        rows = torch.empty(2 * pl[3], m, 2, dtype=torch.float32, device=x.device)  # one partial per column half of a tile
        args.rs_out = rows.data_ptr()
        rowstats["rows"], rowstats["parts"] = rows, 2 * pl[3]
        _keep = rows
    packed, bn = _tiled_s8(args, wgt, taps=1)
    args.wgt, args.block_n, args.wgt_tiled = packed.data_ptr(), bn, 1
    need = int(load().b200sd_gemm_workspace_bytes_s8_linear(C.byref(args)))
    if need:
        ws = _workspace(need, x.device)
        args.workspace = ws.data_ptr()
        args.workspace_bytes = ws.numel() * 4
    _check(load().b200sd_gemm_s8_linear(C.byref(args), _ptr(col_scale), _stream()), "b200sd_gemm_s8_linear")
    return out


def layer_norm_s8(x, gamma, beta, inv_scale, eps=1e-5, out=None):
    """layer_norm (fp16 [rows, c]) whose output is int8: q = clamp(rint(y * inv_scale), -127, 127) of the fp32 y."""
    _req(x, torch.float16, "layer_norm_s8 x")
    rows, c = x.shape
    if out is None:
        out = torch.empty(rows, c, dtype=torch.int8, device=x.device)
    _req(out, torch.int8, "layer_norm_s8 out")
    _check(load().b200sd_layer_norm_s8(_ptr(x), _ptr(gamma), _ptr(beta), float(inv_scale), _ptr(out), rows, c, float(eps),
                                       _stream()), "b200sd_layer_norm_s8")
    return out


def group_norm_s8(x, gamma, beta, groups, eps, inv_scale, silu=True, x1=None, out=None):
    """group_norm (fp16 sources) whose output is int8: q = clamp(rint(y * inv_scale), -127, 127) of the fp32 y."""
    _req(x, torch.float16, "group_norm_s8 x")
    _same16(torch.float16, x1, None, "group_norm_s8 x1")
    nimg, h, w, c0 = x.shape
    c1 = 0 if x1 is None else x1.shape[-1]
    if out is None:
        out = torch.empty(nimg, h, w, c0 + c1, dtype=torch.int8, device=x.device)
    _req(out, torch.int8, "group_norm_s8 out")
    need = int(load().b200sd_group_norm_workspace_bytes(nimg, h * w, c0 + c1, groups))
    ws = _workspace(need, x.device)
    _check(load().b200sd_group_norm_s8(_ptr(x), _ptr(x1), c0, c1, nimg, h * w, groups, float(eps), _ptr(gamma), _ptr(beta),
                                       int(silu), float(inv_scale), _ptr(out), _ptr(ws), ws.numel() * 4, _stream()),
           "b200sd_group_norm_s8")
    return out


def upsample2x_s8(x, inv_scale, out=None):
    """Nearest x2 upsample of fp16 NHWC x into int8: q = clamp(rint(x * inv_scale), -127, 127)."""
    _req(x, torch.float16, "upsample2x_s8 x")
    n, h, w, c = x.shape
    if out is None:
        out = torch.empty(n, 2 * h, 2 * w, c, dtype=torch.int8, device=x.device)
    _req(out, torch.int8, "upsample2x_s8 out")
    _check(load().b200sd_upsample2x_s8(_ptr(x), _ptr(out), n, h, w, c, float(inv_scale), _stream()), "b200sd_upsample2x_s8")
    return out


def absmax(x, slot):
    """slot (fp32 device scalar, >= 0) = max(slot, max |x|) for an fp16 tensor x: the W8A8 calibration probe."""
    _req(x, torch.float16, "absmax x")
    _req(slot, torch.float32, "absmax slot")
    _check(load().b200sd_absmax_f16(_ptr(x), x.numel(), _ptr(slot), _stream()), "b200sd_absmax_f16")
    return slot


def linear_small(x, wgt, bias=None, add=None, act_in=False, act_out=False):
    _req(x, torch.float32, "linear_small x")
    _req(wgt, torch.float16, "linear_small wgt")
    m, k = x.shape
    n = wgt.shape[0]
    out = torch.empty(m, n, dtype=torch.float32, device=x.device)
    _check(load().b200sd_linear_small(_ptr(x), _ptr(wgt), _ptr(bias), _ptr(add), _ptr(out), m, n, k,
                                      int(act_in), int(act_out), _stream()), "b200sd_linear_small")
    return out


def timestep_embedding(t, dim, flip_sin_to_cos=True, freq_shift=0.0):
    _req(t, torch.float32, "timestep_embedding t")
    out = torch.empty(t.shape[0], dim, dtype=torch.float32, device=t.device)
    _check(load().b200sd_timestep_embedding(_ptr(t), _ptr(out), t.shape[0], dim, int(flip_sin_to_cos),
                                            float(freq_shift), _stream()), "b200sd_timestep_embedding")
    return out


def group_norm(x, gamma, beta, groups, eps, silu=False, x1=None, out=None):
    """x NHWC fp16 or bf16 [N, H, W, C0] (optionally ++ x1 [N, H, W, C1], same type) -> normalised [N, H, W, C0+C1]
    in x's type (fp32 statistics either way)."""
    dt = _act_dtype(x, "group_norm x")
    _same16(dt, x1, out, "group_norm x1 / out")
    nimg, h, w, c0 = x.shape
    c1 = 0 if x1 is None else x1.shape[-1]
    if out is None:
        out = torch.empty(nimg, h, w, c0 + c1, dtype=dt, device=x.device)
    need = int(load().b200sd_group_norm_workspace_bytes(nimg, h * w, c0 + c1, groups))
    ws = _workspace(need, x.device)
    name = "b200sd_group_norm" + _sfx(dt)
    _check(getattr(load(), name)(_ptr(x), _ptr(x1), c0, c1, nimg, h * w, groups, float(eps), _ptr(gamma),
                                 _ptr(beta), int(silu), _ptr(out), _ptr(ws), ws.numel() * 4, _stream()), name)
    return out


def group_norm_apply(x, chan0, gamma, beta, groups, eps, silu=False, x1=None, chan1=None, out=None):
    """GroupNorm (+SiLU, + concat) from the producers' per-channel sums ``chan0`` / ``chan1`` [N, C, 2]: no statistics pass."""
    _req(x, torch.float16, "group_norm_apply x")
    nimg, h, w, c0 = x.shape
    c1 = 0 if x1 is None else x1.shape[-1]
    if out is None:
        out = torch.empty(nimg, h, w, c0 + c1, dtype=torch.float16, device=x.device)
    _check(load().b200sd_group_norm_apply(_ptr(x), _ptr(x1), c0, c1, nimg, h * w, groups, float(eps), _ptr(chan0), _ptr(chan1),
                                          _ptr(gamma), _ptr(beta), int(silu), _ptr(out), _stream()), "b200sd_group_norm_apply")
    return out


def layer_norm(x, gamma, beta, eps=1e-5, out=None):
    _req(x, torch.float16, "layer_norm x")
    rows, c = x.shape
    if out is None:
        out = torch.empty_like(x)
    _check(load().b200sd_layer_norm(_ptr(x), _ptr(gamma), _ptr(beta), _ptr(out), rows, c, float(eps), _stream()),
           "b200sd_layer_norm")
    return out


ATTENTION_HEAD_DIMS = (40, 64, 80, 160)  # head dims the attention kernel is built for (include/b200sd.h)


def attention(q, k, v, batch, heads, sq, sk, d=64, mask=None, impl=0, out=None, scale=None, causal=False):
    """q: view [batch*sq, >=heads*d] (row stride = q.stride(0)), k/v: [batch*sk, ...]; out [batch*sq, heads*d].
    d: head dim, one of ATTENTION_HEAD_DIMS.  causal: key j is visible to query i only if j <= i (CLIP text encoder)."""
    for t, nm in ((q, "q"), (k, "k"), (v, "v")):
        if t.dtype != torch.float16 or not t.is_cuda or t.stride(-1) != 1:
            raise B200SDError(f"attention {nm}: expected CUDA fp16 with unit inner stride")
    if out is None:
        out = torch.empty(batch * sq, heads * d, dtype=torch.float16, device=q.device)
    scale = float(d) ** -0.5 if scale is None else float(scale)
    ws = _attention_workspace(q.device, d)
    _check(load().b200sd_attention_ws(_ptr(q), _ptr(k), _ptr(v), _ptr(out), _ptr(mask), batch, heads, sq, sk, d,
                                      q.stride(0), k.stride(0), v.stride(0), out.stride(0), scale,
                                      int(impl) | (0x100 if causal else 0), _ptr(ws), ws.numel(),
                                      _stream()), "b200sd_attention_ws")
    return out


_attn_ws = {}
_attn_ws_retired = []  # outgrown workspaces: graphs captured earlier still point at them


def _attention_workspace(device, d=64):
    """Zero-filled once per device: the stream-K pieces of split query tiles meet here; its counters return to zero at
    the end of every launch.  Launches on one stream are ordered, which is the only way this package launches.
    The partials grow with the head dim d: the buffer is replaced by a larger one the first time a d needs more, except
    during a CUDA-graph capture, where the launch then schedules whole query tiles (engines reserve their largest d when
    they are built, see reserve_attention_workspace)."""
    key = device.index if device.index is not None else torch.cuda.current_device()
    ws = _attn_ws.get(key)
    need = int(load().b200sd_attention_workspace_bytes_for(int(d))) if d != 64 else None
    if ws is None or (need is not None and ws.numel() < need and not torch.cuda.is_current_stream_capturing()):
        size = max(int(load().b200sd_attention_workspace_bytes()), need or 0, 0 if ws is None else ws.numel())
        if ws is not None:
            _attn_ws_retired.append(ws)
        ws = torch.zeros(size, dtype=torch.uint8, device=device)
        _attn_ws[key] = ws
    return ws


def reserve_attention_workspace(device, d):
    """Sizes the device's attention workspace for head dim d (outside any CUDA-graph capture)."""
    return _attention_workspace(torch.device(device), d)


def nchw_to_nhwc(x, c_pad=None, out=None, out_dtype=torch.float16):
    """NCHW fp16 / fp32 -> NHWC out_dtype (fp16 or bf16) with the channels zero padded to c_pad; a given `out`
    decides the type (as in softmax_rows)."""
    n, c, h, w = x.shape
    c_pad = c if c_pad is None else c_pad
    if x.dtype not in (torch.float16, torch.float32) or not x.is_contiguous():
        raise B200SDError("nchw_to_nhwc: expected contiguous fp16/fp32")
    if out is not None:
        out_dtype = out.dtype
    if out_dtype not in ACT_DTYPES:
        raise B200SDError(f"nchw_to_nhwc: out_dtype must be fp16 or bf16, got {out_dtype}")
    if out is None:
        out = torch.empty(n, h, w, c_pad, dtype=out_dtype, device=x.device)
    elif out.dtype != out_dtype or not out.is_contiguous() or tuple(out.shape) != (n, h, w, c_pad):
        raise B200SDError("nchw_to_nhwc: bad output buffer")
    name = "b200sd_nchw_to_nhwc" + _sfx(out_dtype)
    _check(getattr(load(), name)(_ptr(x), int(x.dtype == torch.float32), _ptr(out), n, c, h, w, c_pad, _stream()), name)
    return out


def _f16_or_f32(x, what):
    """Kernels with one fp16 / fp32 input flag: any other type would be read as fp16 bits."""
    if x.dtype not in (torch.float16, torch.float32):
        raise B200SDError(f"{what}: expected fp16 or fp32 input, got {x.dtype}")


def nhwc_to_nchw_f32(x, c=None, out=None):
    _f16_or_f32(x, "nhwc_to_nchw_f32")
    n, h, w, c_pad = x.shape
    c = c_pad if c is None else c
    if out is None:
        out = torch.empty(n, c, h, w, dtype=torch.float32, device=x.device)
    _check(load().b200sd_nhwc_to_nchw_f32(_ptr(x), int(x.dtype == torch.float32), _ptr(out), n, c, h, w, c_pad,
                                          _stream()), "b200sd_nhwc_to_nchw_f32")
    return out


def upsample2x(x, out=None):
    """Nearest x2 upsample of an NHWC fp16 or bf16 tensor (a byte copy: one kernel for both)."""
    dt = _act_dtype(x, "upsample2x x")
    _same16(dt, out, None, "upsample2x out")
    n, h, w, c = x.shape
    if out is None:
        out = torch.empty(n, 2 * h, 2 * w, c, dtype=dt, device=x.device)
    _check(load().b200sd_upsample2x(_ptr(x), _ptr(out), n, h, w, c, _stream()), "b200sd_upsample2x")
    return out


def add(a, b, out=None):
    _req(a, torch.float16, "add a")
    _req(b, torch.float16, "add b")
    if out is None:
        out = torch.empty_like(a)
    _check(load().b200sd_add(_ptr(a), _ptr(b), _ptr(out), a.numel(), _stream()), "b200sd_add")
    return out


MAX_CONTROLNETS = 8  # B200SD_MAX_CONTROLNETS


def control_inject(skip, residuals, scales, out=None):
    """ControlNet residual injection, one launch whatever the number of nets: out = fp16(skip + t) with
    t = fp16(s_0 r_0), t = fp16(t + fp16(s_k r_k)) -- diffusers' fp16 order for conditioning_scale, several ControlNets
    and the UNet's add.  ``skip`` None: out = t.  ``residuals``: fp16 tensors shaped like ``skip``; ``scales``: fp32 CUDA
    tensor [len(residuals)], read by the kernel, so a captured graph replays with the values it holds then."""
    n = len(residuals)
    if not 1 <= n <= MAX_CONTROLNETS:
        raise B200SDError(f"control_inject: {n} residuals, at most {MAX_CONTROLNETS}")
    ref = residuals[0] if skip is None else skip
    _req(ref, torch.float16, "control_inject skip")
    for r in residuals:
        _req(r, torch.float16, "control_inject residual")
        if r.shape != ref.shape:
            raise B200SDError(f"control_inject: residual of shape {tuple(r.shape)}, expected {tuple(ref.shape)}")
    _req(scales, torch.float32, "control_inject scales")
    if scales.numel() < n:
        raise B200SDError(f"control_inject: {scales.numel()} scales for {n} residuals")
    if out is None:
        out = torch.empty_like(ref)
    ptrs = (C.c_void_p * n)(*[r.data_ptr() for r in residuals])
    _check(load().b200sd_control_inject(_ptr(skip), ptrs, _ptr(scales), n, _ptr(out), ref.numel(), _stream()),
           "b200sd_control_inject")
    return out


def embed_tokens(ids, token_embedding, position_embedding, out=None):
    """ids fp32 [B, S]; tables fp16 [V, D] / [S, D] -> fp16 [B*S, D] (token + position embedding)."""
    _req(ids, torch.float32, "embed_tokens ids")
    _req(token_embedding, torch.float16, "embed_tokens token_embedding")
    _req(position_embedding, torch.float16, "embed_tokens position_embedding")
    b, s = ids.shape
    v, d = token_embedding.shape
    if position_embedding.shape[0] < s or position_embedding.shape[1] != d:
        raise B200SDError("embed_tokens: position table does not cover the sequence")
    if out is None:
        out = torch.empty(b * s, d, dtype=torch.float16, device=ids.device)
    _check(load().b200sd_embed_tokens(_ptr(ids), _ptr(token_embedding), _ptr(position_embedding), _ptr(out), b, s, d, v,
                                      _stream()), "b200sd_embed_tokens")
    return out


def ctx_to_tokens(ctx, out=None):
    """(B, D, 1, S) fp16/fp32 -> [B*S, D] fp16."""
    _f16_or_f32(ctx, "ctx_to_tokens")
    b, d, _, s = ctx.shape
    if not ctx.is_contiguous():
        raise B200SDError("ctx_to_tokens: expected contiguous input")
    if out is None:
        out = torch.empty(b * s, d, dtype=torch.float16, device=ctx.device)
    _check(load().b200sd_ctx_to_tokens(_ptr(ctx), int(ctx.dtype == torch.float32), _ptr(out), b, d, s, _stream()),
           "b200sd_ctx_to_tokens")
    return out


def cfg_scheduler_step(noise_pred, latents, coeffs: StepCoeffs, hist=None, denoised=None, unet_in=None):
    _req(noise_pred, torch.float32, "cfg_scheduler_step noise_pred")
    _req(latents, torch.float32, "cfg_scheduler_step latents")
    n, c, h, w = latents.shape
    c_pad = 0 if unet_in is None else unet_in.shape[-1]
    _check(load().b200sd_cfg_scheduler_step(_ptr(noise_pred), _ptr(latents), _ptr(hist), _ptr(denoised),
                                            _ptr(unet_in), c_pad, n, c, h, w, C.byref(coeffs), _stream()),
           "b200sd_cfg_scheduler_step")
    return latents


def cfg_scheduler_step_noised(noise_pred, latents, coeffs: StepCoeffs, noise_scale, key, offset, hist=None,
                              denoised=None, unet_in=None):
    """``cfg_scheduler_step`` plus ``noise_scale * z``, z the Philox normals of ``rng.NvRandomSource(key)``'s
    ``offset``-th draw; ``key``: a one-element int32 / uint32 CUDA tensor holding the key's bits."""
    _req(noise_pred, torch.float32, "cfg_scheduler_step_noised noise_pred")
    _req(latents, torch.float32, "cfg_scheduler_step_noised latents")
    if not (key.is_cuda and key.numel() == 1 and key.element_size() == 4):
        raise B200SDError("cfg_scheduler_step_noised: key must be a one-element 4-byte CUDA tensor")
    n, c, h, w = latents.shape
    c_pad = 0 if unet_in is None else unet_in.shape[-1]
    _check(load().b200sd_cfg_scheduler_step_noised(_ptr(noise_pred), _ptr(latents), _ptr(hist), _ptr(denoised),
                                                   _ptr(unet_in), c_pad, n, c, h, w, C.byref(coeffs), float(noise_scale),
                                                   _ptr(key), int(offset) & 0xFFFFFFFF, _stream()),
           "b200sd_cfg_scheduler_step_noised")
    return latents


def cfg_scheduler_step_blend(noise_pred, latents, coeffs: StepCoeffs, mask, image_latents, noise, a, b,
                             noise_scale=0.0, key=None, offset=0, hist=None, denoised=None, unet_in=None):
    """``cfg_scheduler_step`` (``_noised`` when ``key`` is given), then the inpainting blend
    ``x' = m x' + (1 - m)(a image_latents + b noise)``: ``mask`` fp32 [n, h*w] (or [n, 1, h, w]), ``image_latents`` /
    ``noise`` fp32 like ``latents``."""
    _req(noise_pred, torch.float32, "cfg_scheduler_step_blend noise_pred")
    _req(latents, torch.float32, "cfg_scheduler_step_blend latents")
    n, c, h, w = latents.shape
    _req(mask, torch.float32, "cfg_scheduler_step_blend mask")
    if mask.numel() != n * h * w:
        raise B200SDError(f"cfg_scheduler_step_blend: mask has {mask.numel()} elements, expected {n * h * w}")
    for name, t in (("image_latents", image_latents), ("noise", noise)):
        _req(t, torch.float32, f"cfg_scheduler_step_blend {name}")
        if tuple(t.shape) != (n, c, h, w):
            raise B200SDError(f"cfg_scheduler_step_blend: {name} has shape {tuple(t.shape)}, expected {(n, c, h, w)}")
    if key is not None and not (key.is_cuda and key.numel() == 1 and key.element_size() == 4):
        raise B200SDError("cfg_scheduler_step_blend: key must be a one-element 4-byte CUDA tensor")
    c_pad = 0 if unet_in is None else unet_in.shape[-1]
    args = BlendArgs(_ptr(mask), _ptr(image_latents), _ptr(noise), float(a), float(b))
    _check(load().b200sd_cfg_scheduler_step_blend(_ptr(noise_pred), _ptr(latents), _ptr(hist), _ptr(denoised),
                                                  _ptr(unet_in), c_pad, n, c, h, w, C.byref(coeffs),
                                                  float(noise_scale), _ptr(key), int(offset) & 0xFFFFFFFF,
                                                  C.byref(args), _stream()),
           "b200sd_cfg_scheduler_step_blend")
    return latents


def scheduler_step_guidance_free(noise_pred, latents, coeffs: StepCoeffs, noise_scale=0.0, key=None, offset=0,
                                 blend=None, hist=None, denoised=None, unet_in=None):
    """The step without classifier-free guidance: ``noise_pred`` holds ONE prediction per image (fp32, the size of
    ``latents``; NHWC when ``coeffs.noise_pred_nhwc``), ``unet_in`` receives the next UNet input in its first n rows.
    ``key`` / ``offset``: the ancestral noise of ``cfg_scheduler_step_noised``; ``blend`` = (mask, image_latents,
    noise, a, b): the inpainting blend of ``cfg_scheduler_step_blend``."""
    what = "scheduler_step_guidance_free"
    _req(noise_pred, torch.float32, f"{what} noise_pred")
    _req(latents, torch.float32, f"{what} latents")
    n, c, h, w = latents.shape
    if noise_pred.numel() != latents.numel():
        raise B200SDError(f"{what}: noise_pred has {noise_pred.numel()} elements, expected one prediction per image "
                          f"({latents.numel()})")
    if key is not None and not (key.is_cuda and key.numel() == 1 and key.element_size() == 4):
        raise B200SDError(f"{what}: key must be a one-element 4-byte CUDA tensor")
    args = None
    if blend is not None:
        mask, image_latents, noise, a, b = blend
        _req(mask, torch.float32, f"{what} mask")
        if mask.numel() != n * h * w:
            raise B200SDError(f"{what}: mask has {mask.numel()} elements, expected {n * h * w}")
        for name, t in (("image_latents", image_latents), ("noise", noise)):
            _req(t, torch.float32, f"{what} {name}")
            if tuple(t.shape) != (n, c, h, w):
                raise B200SDError(f"{what}: {name} has shape {tuple(t.shape)}, expected {(n, c, h, w)}")
        args = BlendArgs(_ptr(mask), _ptr(image_latents), _ptr(noise), float(a), float(b))
    if unet_in is not None and unet_in.shape[0] < n:
        raise B200SDError(f"{what}: unet_in has {unet_in.shape[0]} rows, expected at least {n}")
    c_pad = 0 if unet_in is None else unet_in.shape[-1]
    _check(load().b200sd_scheduler_step_guidance_free(_ptr(noise_pred), _ptr(latents), _ptr(hist), _ptr(denoised),
                                                      _ptr(unet_in), c_pad, n, c, h, w, C.byref(coeffs),
                                                      float(noise_scale), _ptr(key), int(offset) & 0xFFFFFFFF,
                                                      None if args is None else C.byref(args), _stream()),
           "b200sd_scheduler_step_guidance_free")
    return latents


def image_postprocess(x, c=3, want_u8=False):
    _f16_or_f32(x, "image_postprocess")
    n, h, w, c_pad = x.shape
    of = torch.empty(n, h, w, c, dtype=torch.float32, device=x.device)
    ou = torch.empty(n, h, w, c, dtype=torch.uint8, device=x.device) if want_u8 else None
    _check(load().b200sd_image_postprocess(_ptr(x), int(x.dtype == torch.float32), c_pad, _ptr(of), _ptr(ou), n, h,
                                           w, c, _stream()), "b200sd_image_postprocess")
    return (of, ou) if want_u8 else of


def clip_preprocess(images_u8, h_table, v_table, mean, std, out=None, tmp=None):
    """u8 NHWC [n, h, w, 3] -> fp32 NCHW pixel_values [n, 3, crop_h, crop_w]: Pillow BICUBIC resize (horizontal then
    vertical fixed-point pass), centre crop, rescale, normalise.  h_table / v_table: (bounds int32 [crop, 2], coeffs
    int32 [crop, ksize]) CUDA tensors from ``safety_checker.resample_table`` restricted to the crop window."""
    _req(images_u8, torch.uint8, "clip_preprocess images")
    n, h, w, c = images_u8.shape
    if c != 3:
        raise B200SDError(f"clip_preprocess: expected 3 channels, got {c}")
    (hb, hc), (vb, vc) = h_table, v_table
    for t, nm in ((hb, "h bounds"), (hc, "h coeffs"), (vb, "v bounds"), (vc, "v coeffs")):
        _req(t, torch.int32, f"clip_preprocess {nm}")
    crop_w, crop_h = hb.shape[0], vb.shape[0]
    if out is None:
        out = torch.empty(n, 3, crop_h, crop_w, dtype=torch.float32, device=images_u8.device)
    _req(out, torch.float32, "clip_preprocess out")
    if tmp is None or tmp.numel() < n * h * crop_w * 3:
        tmp = torch.empty(n * h * crop_w * 3, dtype=torch.uint8, device=images_u8.device)
    fm, fs = (C.c_float * 3)(*[float(v) for v in mean]), (C.c_float * 3)(*[float(v) for v in std])
    _check(load().b200sd_clip_preprocess(_ptr(images_u8), n, h, w, _ptr(tmp), _ptr(hb), _ptr(hc), hc.shape[1],
                                         _ptr(vb), _ptr(vc), vc.shape[1], crop_h, crop_w, fm, fs, _ptr(out),
                                         _stream()), "b200sd_clip_preprocess")
    return out


def patchify(pixel_values, patch, k_pad, out=None):
    """fp32 NCHW [n, c, S, S] -> fp16 [n * (1 + (S/patch)^2), k_pad]: per image a zero class-token row, then the
    patches in row-major order, each flattened in (channel, ky, kx) order and zero padded to k_pad columns."""
    _req(pixel_values, torch.float32, "patchify pixel_values")
    n, c, s, s2 = pixel_values.shape
    if s != s2 or s % patch:
        raise B200SDError(f"patchify: {s}x{s2} images do not tile into {patch}x{patch} patches")
    rows = n * (1 + (s // patch) ** 2)
    if out is None:
        out = torch.empty(rows, k_pad, dtype=torch.float16, device=pixel_values.device)
    _req(out, torch.float16, "patchify out")
    if tuple(out.shape) != (rows, k_pad):
        raise B200SDError(f"patchify: out has shape {tuple(out.shape)}, expected {(rows, k_pad)}")
    _check(load().b200sd_patchify(_ptr(pixel_values), n, c, s, patch, k_pad, _ptr(out), _stream()), "b200sd_patchify")
    return out


def safety_concepts(image_embeds, concepts, concept_weights, special, special_weights, adjustment=None):
    """fp32 image_embeds [n, dim] -> (concept_scores fp32 [n, n_concepts], has_nsfw fp32 [n]) against the
    L2-normalised concept tables; ``adjustment``: a one-element fp32 CUDA tensor (None: 0)."""
    for t, nm in ((image_embeds, "image_embeds"), (concepts, "concepts"), (concept_weights, "concept_weights"),
                  (special, "special"), (special_weights, "special_weights")):
        _req(t, torch.float32, f"safety_concepts {nm}")
    if adjustment is not None:
        _req(adjustment, torch.float32, "safety_concepts adjustment")
    n, dim = image_embeds.shape
    nc, ns = concepts.shape[0], special.shape[0]
    if concepts.shape[1] != dim or special.shape[1] != dim:
        raise B200SDError(f"safety_concepts: concept tables of width {concepts.shape[1]} / {special.shape[1]}, "
                          f"embeddings of width {dim}")
    scores = torch.empty(n, nc, dtype=torch.float32, device=image_embeds.device)
    flags = torch.empty(n, dtype=torch.float32, device=image_embeds.device)
    _check(load().b200sd_safety_concepts(_ptr(image_embeds), n, dim, _ptr(concepts), _ptr(concept_weights), nc,
                                         _ptr(special), _ptr(special_weights), ns, _ptr(adjustment), _ptr(scores),
                                         _ptr(flags), _stream()), "b200sd_safety_concepts")
    return scores, flags


def filter_images(has_nsfw, images=None, images_u8=None):
    """Zero, in place, every image whose ``has_nsfw`` entry (fp32 [n]) is non-zero: fp32 and / or u8 NHWC images."""
    _req(has_nsfw, torch.float32, "filter_images has_nsfw")
    ref = images if images is not None else images_u8
    if ref is None:
        raise B200SDError("filter_images: no images given")
    if images is not None:
        _req(images, torch.float32, "filter_images images")
    if images_u8 is not None:
        _req(images_u8, torch.uint8, "filter_images images_u8")
        if images is not None and images_u8.shape != images.shape:
            raise B200SDError("filter_images: the fp32 and u8 images differ in shape")
    n, h, w, c = ref.shape
    if has_nsfw.numel() != n:
        raise B200SDError(f"filter_images: {has_nsfw.numel()} flags for {n} images")
    _check(load().b200sd_filter_images(_ptr(has_nsfw), _ptr(images), _ptr(images_u8), n, h, w, c, _stream()),
           "b200sd_filter_images")
    return images, images_u8


def softmax_rows(scores, scale, out=None, out_dtype=torch.float16):
    """fp32 scores [rows, cols] -> probabilities in out_dtype (fp16 or bf16: the type of the P V GEMM)."""
    _req(scores, torch.float32, "softmax_rows scores")
    rows, cols = scores.shape
    if out is not None:
        out_dtype = out.dtype
    if out_dtype not in ACT_DTYPES:
        raise B200SDError(f"softmax_rows: out_dtype must be fp16 or bf16, got {out_dtype}")
    if out is None:
        out = torch.empty(rows, cols, dtype=out_dtype, device=scores.device)
    name = "b200sd_softmax_rows" + _sfx(out_dtype)
    _check(getattr(load(), name)(_ptr(scores), _ptr(out), rows, cols, float(scale), _stream()), name)
    return out


def latent_prep(z, w, b, inv_scale, c_pad=8, out_dtype=torch.float16):
    """fp32 NCHW latents -> post_quant_conv(z * inv_scale) as NHWC out_dtype (fp16 or bf16), c_pad channels."""
    _req(z, torch.float32, "latent_prep z")
    if out_dtype not in ACT_DTYPES:
        raise B200SDError(f"latent_prep: out_dtype must be fp16 or bf16, got {out_dtype}")
    n, c, h, wd = z.shape
    out = torch.empty(n, h, wd, c_pad, dtype=out_dtype, device=z.device)
    name = "b200sd_latent_prep" + _sfx(out_dtype)
    _check(getattr(load(), name)(_ptr(z), _ptr(w), _ptr(b), float(inv_scale), _ptr(out), n, c, h, wd, c_pad, _stream()),
           name)
    return out
