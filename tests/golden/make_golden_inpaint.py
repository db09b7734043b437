"""Golden fixtures for 9-channel inpainting UNets (runwayml/stable-diffusion-inpainting,
stabilityai/stable-diffusion-2-inpainting: ``"in_channels": 9``), produced by the UNMODIFIED reference UNet through
oracle/ref_unet.py on the CPU in fp32.  Build container only:

    python tests/golden/make_golden_inpaint.py

Writes
  unet_tiny_inpaint.npz   config.TINY_UNET with in_channels = 9, 16x16 latents, ORIGINAL
  unet_sd15_inpaint.npz   config.SD15_UNET with in_channels = 9, 64x64 latents, ORIGINAL
Weights are regenerated from the seed on the test side (see make_golden.py).
"""
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)

from b200sd import config  # noqa: E402
from oracle import ref_unet  # noqa: E402
from make_golden import fingerprint, unet_inputs  # noqa: E402

OUT = os.path.dirname(os.path.abspath(__file__))
TINY_INPAINT = dict(config.TINY_UNET, in_channels=9)
SD15_INPAINT = dict(config.SD15_UNET, in_channels=9)


def main():
    torch.manual_seed(0)
    for name, cfg, wseed, iseed, t in [("tiny_inpaint", TINY_INPAINT, 61, 62, 981.0),
                                       ("sd15_inpaint", SD15_INPAINT, 63, 64, 501.0)]:
        sd = config.random_state_dict(config.unet_param_shapes(cfg), seed=wseed)
        x, c = unet_inputs(cfg, iseed)
        m = ref_unet.build_unet(cfg, sd, impl="ORIGINAL")
        with torch.no_grad():
            out = m(x, torch.tensor([t, t]), c)[0].numpy()
        del m
        np.savez_compressed(os.path.join(OUT, f"unet_{name}.npz"), weight_seed=wseed, input_seed=iseed,
                            timestep=t, fingerprint=fingerprint(sd), noise_pred_ORIGINAL=out.astype(np.float32))
        print(name, out.shape, float(np.abs(out).max()))


if __name__ == "__main__":
    main()
