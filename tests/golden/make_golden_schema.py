"""Writes tests/golden/schema_tiny_live.npz: what test_oracle.py compares against the UNMODIFIED reference modules
(python_coreml_stable_diffusion.{unet,controlnet}, imported through oracle/ref_unet.py), stored so the comparison runs
without the reference tree:
  * sha256 of the parameter schema (sorted "name shape" lines) of every UNet / ControlNet configuration the project
    builds, as the reference modules construct it;
  * the tiny UNet's output for each attention implementation (weights seed 7, inputs seed 8, t = [501, 21]).
Run where the reference tree is present:

    python tests/golden/make_golden_schema.py
"""
import hashlib
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

from b200sd import config  # noqa: E402
from oracle import ref_unet  # noqa: E402


def schema_digest(shapes):
    lines = "\n".join(f"{k} {tuple(int(d) for d in v)}" for k, v in sorted(shapes.items()))
    return hashlib.sha256(lines.encode()).hexdigest()


def main():
    assert ref_unet.available(), "reference tree not importable"
    out = {}
    for name, cfg, xl in (("TINY_UNET", config.TINY_UNET, False), ("SD21_BASE_UNET", config.SD21_BASE_UNET, False),
                          ("SDXL_BASE_UNET", config.SDXL_BASE_UNET, True)):
        with torch.device("meta"):
            m = ref_unet.build_unet(cfg, None, xl=xl)
        out[f"schema_{name}"] = np.array(schema_digest({k: v.shape for k, v in m.state_dict().items()}))
    for name, cfg in (("TINY_CONTROLNET", config.TINY_CONTROLNET), ("SD21_CONTROLNET", config.SD21_CONTROLNET)):
        with torch.device("meta"):
            m = ref_unet.build_controlnet(cfg)
        out[f"schema_{name}"] = np.array(schema_digest({k: v.shape for k, v in m.state_dict().items()}))
    cfg = config.TINY_UNET
    sd = config.random_state_dict(config.unet_param_shapes(cfg), seed=7)
    g = torch.Generator().manual_seed(8)  # the inputs test_oracle._inputs(cfg, 8) draws
    x = torch.randn(2, cfg["in_channels"], cfg["sample_size"], cfg["sample_size"], generator=g)
    c = torch.randn(2, cfg["cross_attention_dim"], 1, 77, generator=g)
    t = torch.tensor([501.0, 21.0])
    with torch.no_grad():
        for impl in ("ORIGINAL", "SPLIT_EINSUM", "SPLIT_EINSUM_V2"):
            out[f"tiny_{impl}"] = ref_unet.build_unet(cfg, sd, impl=impl)(x, t, c)[0].numpy()
    np.savez_compressed(os.path.join(os.path.dirname(os.path.abspath(__file__)), "schema_tiny_live.npz"), **out)


if __name__ == "__main__":
    main()
