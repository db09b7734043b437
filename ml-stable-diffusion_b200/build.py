"""In-tree build of ``libb200sd.so`` (sm_90a only) with nvcc.  No JIT cache, no torch extension:
the library is a plain C-ABI shared object (``include/b200sd.h``) loaded with ctypes."""
from __future__ import annotations

import hashlib
import os
import shutil
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
LIB = os.path.join(HERE, "libb200sd.so")
STAMP = os.path.join(HERE, ".libb200sd.stamp")
SOURCES = ["runtime.cu", "gemm_conv.cu", "attention.cu", "norm.cu", "elementwise.cu", "model.cu"]
NVCC_FLAGS = [
    "-gencode", "arch=compute_90a,code=sm_90a", "-lineinfo", "-O3", "-std=c++17",
    "-Xcompiler", "-fPIC", "--use_fast_math_placeholder",
]


def _nvcc():
    for c in (os.environ.get("NVCC"), shutil.which("nvcc"), "/usr/local/cuda/bin/nvcc"):
        if c and os.path.exists(c):
            return c
    raise RuntimeError("nvcc not found")


def _digest():
    h = hashlib.sha256()
    files = [os.path.join(CSRC, f) for f in sorted(os.listdir(CSRC))]
    files.append(os.path.join(os.path.dirname(HERE), "include", "b200sd.h"))
    for f in files:
        with open(f, "rb") as fh:
            h.update(f.encode())
            h.update(fh.read())
    return h.hexdigest()


def build(force: bool = False, verbose: bool = False) -> str:
    """Compile every CUDA source for sm_90a and link ``libb200sd.so``.  Returns its path."""
    dig = _digest()
    if not force and os.path.exists(LIB) and os.path.exists(STAMP):
        with open(STAMP) as f:
            if f.read().strip() == dig:
                return LIB
    nvcc = _nvcc()
    flags = [f for f in NVCC_FLAGS if f != "--use_fast_math_placeholder"]
    objs = []
    procs = []
    build_dir = os.path.join(HERE, "build")
    os.makedirs(build_dir, exist_ok=True)
    for src in SOURCES:
        obj = os.path.join(build_dir, src.replace(".cu", ".o"))
        cmd = [nvcc, *flags, "-c", os.path.join(CSRC, src), "-o", obj]
        if verbose:
            print(" ".join(cmd), file=sys.stderr)
        procs.append((src, subprocess.Popen(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)))
        objs.append(obj)
    for src, p in procs:
        out, _ = p.communicate()
        if p.returncode != 0:
            raise RuntimeError(f"nvcc failed on {src}:\n{out}")
        if verbose and out.strip():
            print(out, file=sys.stderr)
    cmd = [nvcc, "-shared", "-gencode", "arch=compute_90a,code=sm_90a", "-o", LIB, *objs]
    r = subprocess.run(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
    if r.returncode != 0:
        raise RuntimeError(f"link failed:\n{r.stdout}")
    with open(STAMP, "w") as f:
        f.write(dig)
    return LIB


if __name__ == "__main__":
    print(build(force="--force" in sys.argv, verbose=True))
