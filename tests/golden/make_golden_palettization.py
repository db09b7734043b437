"""Golden fixture for palettization.palettizable_layers: the eligible layers of SD-2.1-base, SD-1.5 and SDXL-base by the
reference's rule (``mixed_bit_compression_pre_analysis.get_palettizable_modules``: every nn.Linear / nn.Conv2d whose
weight has more than 1e5 elements), read from the module names of the UNMODIFIED reference UNet.  These names are the
keys of the published recipe JSONs.  The networks are built on the meta device (no weights are allocated).  Build
container only:

    python tests/golden/make_golden_palettization.py
"""
import json
import os
import sys

import torch
import torch.nn as nn

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)

from b200sd import config  # noqa: E402
from oracle import ref_unet  # noqa: E402

OUT = os.path.join(os.path.dirname(os.path.abspath(__file__)), "palettizable_layers.json")
MIN_SIZE = 1e5  # PALETTIZE_MIN_SIZE of the reference


def layers(cfg, xl):
    with torch.device("meta"):
        m = ref_unet.build_unet(cfg, xl=xl)
    return {name: mod.weight.numel() for name, mod in m.named_modules()
            if isinstance(mod, (nn.Linear, nn.Conv2d)) and mod.weight.numel() > MIN_SIZE}


def main():
    out = {"sd21_base": layers(config.SD21_BASE_UNET, False), "sd15": layers(config.SD15_UNET, False),
           "sdxl_base": layers(config.SDXL_BASE_UNET, True)}
    with open(OUT, "w") as f:
        json.dump(out, f, indent=0)
    for k, v in out.items():
        print(k, len(v), "layers,", sum(v.values()) / 1e6, "M parameters")


if __name__ == "__main__":
    main()
