"""CPU tests of the drop-in boundary: the C-ABI library builds/loads and exports every symbol that
include/b200sd.h declares (no compute calls without a GPU), the host-side mirrors validate inputs like
the reference, and the product never imports the oracle."""
import ctypes
import os
import re

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_library_exports_every_declared_symbol():
    import __graft_entry__ as ge
    from b200sd import lib

    ge.build()  # nvcc cross-compiles for sm_90a without a GPU
    hdr = open(os.path.join(ROOT, "include", "b200sd.h")).read()
    declared = set(re.findall(r"\b(b200sd_[a-z0-9_]+)\s*\(", hdr))
    assert len(declared) >= 18
    dll = ctypes.CDLL(lib.lib_path())
    for name in sorted(declared):
        assert hasattr(dll, name), f"{name} declared in b200sd.h but not exported"
    assert declared == set(lib.EXPORTED_SYMBOLS), declared ^ set(lib.EXPORTED_SYMBOLS)
    l = lib.load()
    assert l.b200sd_version() >= 1
    assert isinstance(l.b200sd_last_error(), bytes)


def test_struct_layouts_match_header(tmp_path):
    """sizeof / offsetof of the C-ABI structs as gcc sees include/b200sd.h == the ctypes mirrors in lib.py."""
    import shutil
    import subprocess

    from b200sd import capi, lib
    gcc = shutil.which("gcc")
    if gcc is None:
        pytest.skip("gcc not available")
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    fields_g = [f[0] for f in lib.GemmArgs._fields_]
    fields_s = [f[0] for f in lib.StepCoeffs._fields_]
    fields_u = [f[0] for f in capi.UNetConfig._fields_]
    fields_w = [f[0] for f in capi.Weight._fields_]
    src = ['#include <stdio.h>', '#include <stddef.h>', '#include "b200sd.h"', 'int main(void) {',
           'printf("%zu\\n", sizeof(b200sd_gemm_args));']
    src += [f'printf("%zu\\n", offsetof(b200sd_gemm_args, {f}));' for f in fields_g]
    src += ['printf("%zu\\n", sizeof(b200sd_step_coeffs));']
    src += [f'printf("%zu\\n", offsetof(b200sd_step_coeffs, {f}));' for f in fields_s]
    src += ['printf("%zu\\n", sizeof(b200sd_unet_config));']
    src += [f'printf("%zu\\n", offsetof(b200sd_unet_config, {f}));' for f in fields_u]
    src += ['printf("%zu\\n", sizeof(b200sd_weight));']
    src += [f'printf("%zu\\n", offsetof(b200sd_weight, {f}));' for f in fields_w]
    src += ['return 0; }']
    c = tmp_path / "layout.c"
    c.write_text("\n".join(src))
    exe = tmp_path / "layout"
    subprocess.run([gcc, "-I", os.path.join(root, "include"), str(c), "-o", str(exe)], check=True)
    vals = [int(v) for v in subprocess.run([str(exe)], capture_output=True, text=True, check=True).stdout.split()]
    want = [ctypes.sizeof(lib.GemmArgs)] + [getattr(lib.GemmArgs, f).offset for f in fields_g]
    want += [ctypes.sizeof(lib.StepCoeffs)] + [getattr(lib.StepCoeffs, f).offset for f in fields_s]
    want += [ctypes.sizeof(capi.UNetConfig)] + [getattr(capi.UNetConfig, f).offset for f in fields_u]
    want += [ctypes.sizeof(capi.Weight)] + [getattr(capi.Weight, f).offset for f in fields_w]
    assert vals == want


def test_sass_contains_hopper_tensor_and_tma_instructions():
    """The shipped library must contain warpgroup MMA (HGMMA) and TMA (UTMALDG) SASS, and no legacy mma.sync."""
    import shutil
    import subprocess

    from b200sd import lib
    cuobjdump = shutil.which("cuobjdump") or "/usr/local/cuda/bin/cuobjdump"
    if not os.path.exists(cuobjdump):
        pytest.skip("cuobjdump not available")
    sass = subprocess.run([cuobjdump, "-sass", lib.lib_path()], capture_output=True, text=True).stdout
    assert "sm_90a" in sass
    for mnemonic in ("HGMMA", "UTMALDG"):
        assert mnemonic in sass, mnemonic
    assert "HMMA." not in sass.replace("HGMMA.", ""), "legacy mma.sync path found"


def test_model_boundary_validation_matches_reference_contract():
    """coreml_model.py:97-116: TypeError for non-ndarray / dtype / shape, ValueError for unknown kwarg."""
    from b200sd.model import B200Model

    m = B200Model({"sample": {"shape": (2, 4, 64, 64), "dtype": np.dtype(np.float16)}}, "cpu")
    m._verify_inputs(sample=np.zeros((2, 4, 64, 64), np.float16))
    with pytest.raises(TypeError):
        m._verify_inputs(sample=np.zeros((2, 4, 64, 64), np.float32))
    with pytest.raises(TypeError):
        m._verify_inputs(sample=np.zeros((1, 4, 64, 64), np.float16))
    with pytest.raises(TypeError):
        m._verify_inputs(sample=[0.0])
    with pytest.raises(ValueError):
        m._verify_inputs(latents=np.zeros(1, np.float16))


def test_missing_library_fails_loudly(tmp_path, monkeypatch):
    from b200sd import lib

    monkeypatch.setattr(lib, "_lib", None)
    monkeypatch.setattr(lib, "_LIB_PATH", str(tmp_path / "nope.so"))
    with pytest.raises(lib.B200SDError, match="no CPU or PyTorch fallback"):
        lib.load()


def test_product_never_imports_the_oracle():
    pkg = os.path.join(ROOT, "ml-stable-diffusion_b200")
    for dirpath, _, files in os.walk(pkg):
        for f in files:
            if f.endswith((".py", ".cu", ".cuh", ".h")):
                src = open(os.path.join(dirpath, f)).read()
                assert not re.search(r"^\s*(from|import)\s+oracle\b", src, re.M), f


def test_attention_switch_and_scheduler_map_surface():
    from b200sd import unet, scheduler

    assert [e.value for e in unet.AttentionImplementations] == ["ORIGINAL", "SPLIT_EINSUM", "SPLIT_EINSUM_V2"]
    assert unet.ATTENTION_IMPLEMENTATION_IN_EFFECT is unet.AttentionImplementations.SPLIT_EINSUM  # unet.py:39
    assert {"DDIM", "PNDM", "DPMSolverMultistep"} <= set(scheduler.SCHEDULER_MAP)


def test_synthetic_text_path_shapes():
    from b200sd.pipeline import SyntheticTextEncoder, SyntheticTokenizer

    ids = SyntheticTokenizer()("a high quality photo of an astronaut riding a horse in space")
    assert ids.shape == (1, 77) and ids.dtype == np.float32 and ids[0, 0] == 49406 and ids[0, -1] == 49407
    out = SyntheticTextEncoder(1024)(input_ids=ids)["last_hidden_state"]
    assert out.shape == (1, 77, 1024)
    assert np.array_equal(out, SyntheticTextEncoder(1024)(input_ids=ids)["last_hidden_state"])


def test_gemm_planner_invariants_over_unet_shapes():
    """Host-only: the tiling plan for every conv / linear shape class of SD-2.1-base and SDXL-base (batch 2)
    satisfies the constraints the kernels rely on (no GPU needed: b200sd_gemm_describe_plan)."""
    import re

    from b200sd import lib

    shapes = []
    for hw, chans in ((64, (320, 640, 960)), (32, (320, 640, 960, 1280, 1920)), (16, (640, 1280, 1920, 2560)),
                      (8, (1280, 2560)), (96, (320, 640, 960)), (48, (320, 640, 1280, 1920)), (24, (640, 1280, 2560))):
        for cin in chans:
            for cout in (320, 640, 1280):
                shapes.append(dict(mode=1, n=cout, c0=cin, n_img=2, h=hw, w=hw, bias_rows=hw * hw))
                shapes.append(dict(mode=1, n=cout, c0=cin, n_img=2, h=hw, w=hw, has_residual=True))
        for c in (320, 640, 1280):
            m = 2 * hw * hw
            shapes += [dict(mode=0, m=m, n=3 * c, c0=c, has_bias=False), dict(mode=0, m=m, n=c, c0=c, has_residual=True),
                       dict(mode=0, m=m, n=8 * c, c0=c, geglu=True), dict(mode=0, m=m, n=c, c0=4 * c, has_residual=True)]
    shapes += [dict(mode=0, m=154, n=2560, c0=1024, has_bias=False), dict(mode=0, m=154, n=640, c0=2048, has_bias=False)]
    for kw in shapes:
        plan = lib.describe_plan(**kw)
        f = {k: int(v) for k, v in re.findall(r"(\w+)=(-?\d+)(?:\s|$)", plan)}
        bn, splits, stages, kb = f["block_n"], f["splits"], f["stages"], f["kb_total"]
        assert bn % 16 == 0 and 16 <= bn <= 256 and 2 <= stages <= 8, plan
        assert f["n_tiles"] * bn >= f["N"] and (f["n_tiles"] - 1) * bn < f["N"], plan
        assert 1 <= splits <= kb, plan
        if kw.get("geglu"):
            assert splits == 1, plan
        per_stage = 16384 + bn * 128
        assert stages * per_stage + f["epi_smem"] <= 220 * 1024, plan
        if f["cluster"]:
            assert splits in (2, 4, 8) and bn % 32 == 0 and 512 * (bn + 4) <= stages * per_stage, plan


def test_sdxl_prompt_encoding_follows_the_reference_branch():
    """pipeline.py:123-257 (xl): hidden_embeds of both encoders concatenated on the feature axis, pooled output of the
    last encoder, zero negatives by default, uncond half first.  Host logic only (stub encoders, no GPU)."""
    import types

    from b200sd.pipeline import B200StableDiffusionPipeline as P

    def enc(d, p, scale):
        def call(input_ids):
            s = float(np.asarray(input_ids).sum())
            return {"hidden_embeds": np.full((1, 77, d), scale * s, np.float32),
                    "pooled_outputs": np.full((1, p), -scale * s, np.float32)}
        return call

    tok = lambda text: np.full((1, 77), float(len(text)), np.float32)  # noqa: E731
    stub = types.SimpleNamespace(tokenizer=tok, tokenizer_2=tok, text_encoder=enc(6, 3, 1.0), text_encoder_2=enc(10, 5, 2.0),
                                 force_zeros_for_empty_prompt=True)
    emb, pooled = P._encode_prompt_xl(stub, ["ab", "abcd"], True)
    assert emb.shape == (4, 16, 1, 77) and emb.dtype == np.float16 and pooled.shape == (4, 5)
    assert not emb[:2].any() and not pooled[:2].any()                      # zero negatives, uncond half first
    assert emb[2, 0, 0, 0] == 2 * 77 and emb[2, 6, 0, 0] == 2 * 2 * 77    # encoder 1 features first, then encoder 2
    assert pooled[3, 0] == -2.0 * 4 * 77                                   # pooled output of the LAST encoder
    emb2, pooled2 = P._encode_prompt_xl(stub, ["ab"], True, negative_prompt="xyz")
    assert emb2.shape == (2, 16, 1, 77) and emb2[0, 0, 0, 0] == 3 * 77 and pooled2[0, 0] == -2.0 * 3 * 77
    refiner = types.SimpleNamespace(tokenizer=None, tokenizer_2=tok, text_encoder=None, text_encoder_2=enc(10, 5, 2.0),
                                    force_zeros_for_empty_prompt=True)
    emb3, pooled3 = P._encode_prompt_xl(refiner, ["ab"], False)
    # without guidance both batch halves of the UNet carry the prompt (the engine always runs 2B rows)
    assert emb3.shape == (2, 10, 1, 77) and pooled3.shape == (2, 5) and np.array_equal(emb3[0], emb3[1])
    with pytest.raises(ValueError, match="batch size"):
        P._encode_prompt_xl(stub, ["ab", "cd"], True, negative_prompt=["x"])


def test_bench_refuses_to_run_the_product_arm_without_a_gpu():
    """bench.py has no CPU fallback for the product arm: without a CUDA device it prints an error line and exits 1
    (the CPU numbers come from `--impl reference` only)."""
    import json
    import subprocess
    import sys

    import torch
    if torch.cuda.is_available():
        pytest.skip("a GPU is present")
    r = subprocess.run([sys.executable, os.path.join(ROOT, "bench.py"), "--steps", "1", "--warmup", "1"],
                       capture_output=True, text=True, timeout=300)
    assert r.returncode == 1
    line = json.loads(r.stdout.strip().splitlines()[-1])
    assert "no CUDA device" in line["error"] and "--impl reference" in line["error"]


def test_every_kernel_waits_for_its_grid_dependency():
    """Programmatic dependent launch is on by default, so EVERY kernel of the library must execute griddepcontrol.wait
    (`pdl_wait()`) before it touches global memory.  Source scan: cheap guard against a new kernel forgetting it."""
    csrc = os.path.join(ROOT, "ml-stable-diffusion_b200", "csrc")
    seen = 0
    for f in sorted(os.listdir(csrc)):
        if not f.endswith(".cu"):
            continue
        src = open(os.path.join(csrc, f)).read()
        for m in re.finditer(r"__global__[^{;]*\{", src):
            end = src.find("\n}\n", m.end())
            body = src[m.end():end]
            seen += 1
            assert "pdl_wait()" in body, f"{f}: kernel at offset {m.start()} never calls pdl_wait()"
    assert seen >= 20
