import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (H100); run with -m gpu")


def pytest_sessionstart(session):
    """Test convenience only: a fresh checkout has no libb200sd.so (build artefacts are not in git).  If nvcc is
    here, build it once so the boundary tests (dlopen + exported symbols + SASS check) can run; the product itself
    never builds or falls back on its own -- lib.load() raises when the library is missing."""
    import shutil

    lib = os.path.join(ROOT, "ml-stable-diffusion_b200", "libb200sd.so")
    if not os.path.exists(lib) and (shutil.which("nvcc") or os.path.exists("/usr/local/cuda/bin/nvcc")):
        import importlib.util
        spec = importlib.util.spec_from_file_location("_b200sd_build", os.path.join(ROOT, "ml-stable-diffusion_b200", "build.py"))
        mod = importlib.util.module_from_spec(spec)
        spec.loader.exec_module(mod)
        mod.build()


@pytest.fixture(scope="session")
def cuda_lib():
    import torch

    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    # the PyTorch fp32 reference ops must not depend on cuDNN/TF32: loading cuDNN on a fresh box can take
    # minutes (observed) and TF32 would blur the comparison
    torch.backends.cudnn.enabled = False
    torch.backends.cuda.matmul.allow_tf32 = False
    torch.backends.cudnn.allow_tf32 = False
    from b200sd import lib

    lib.load()  # raises loudly if libb200sd.so is missing -- never fall back
    return lib
