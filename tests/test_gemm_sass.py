"""CPU test of the GEMM kernel's machine code: ptxas must keep the wgmma pipeline of every wgmma_gemm_kernel
instantiation (one k-block in flight behind the one being issued) and must not spill its accumulators."""
import os
import re
import shutil
import subprocess

import pytest


def _sass_functions(path):
    cuobjdump = shutil.which("cuobjdump") or "/usr/local/cuda/bin/cuobjdump"
    if not os.path.exists(cuobjdump):
        pytest.skip("cuobjdump not available")
    sass = subprocess.run([cuobjdump, "-sass", path], capture_output=True, text=True, check=True).stdout
    for chunk in re.split(r"\n\s*Function : ", sass)[1:]:
        name, body = chunk.split("\n", 1)
        yield name.strip(), body


def test_gemm_kernels_pipeline_wgmma_and_do_not_spill():
    import __graft_entry__ as ge
    from b200sd import lib

    ge.build()
    kernels = {name: body for name, body in _sass_functions(lib.lib_path()) if "wgmma_gemm_kernel" in name}
    assert len(kernels) >= 8, sorted(kernels)
    for name, body in kernels.items():
        hgmma = len(re.findall(r"\bHGMMA\.", body))
        wait0 = len(re.findall(r"WARPGROUP\.DEPBAR\.LE gsb0, 0x0\b", body))
        wait_n = len(re.findall(r"WARPGROUP\.DEPBAR\.LE gsb0, 0x[1-9a-f]", body))
        assert hgmma > 0, name
        # serialised wgmma: ptxas puts a wait-for-all after every HGMMA and never waits with a non-zero count
        assert wait_n >= 1 and wait0 <= 2, f"{name}: {hgmma} HGMMA, {wait0} waits for 0, {wait_n} waits for > 0"
        spills = re.findall(r"\b(LDL|STL)(\.\w+)*\b", body)
        assert not spills, f"{name}: {len(spills)} local-memory (spill) instructions"
