"""Golden fixture for Stable Diffusion 2.0 / 2.1 768-v (config.SD21_UNET: the SD-2.1-base UNet at 96x96 latents),
produced by the UNMODIFIED reference UNet (python_coreml_stable_diffusion.unet) through oracle/ref_unet.py on the CPU in
fp32, ORIGINAL attention.  Level-0 self-attention runs over 9216 tokens here: the (2, 5, 9216, 9216) fp32 score tensor
alone is 3.4 GB.  Build container only:

    python tests/golden/make_golden_sd21_768.py

Writes unet_sd21_768.npz (seeds, timestep, weight fingerprint, output); weights are regenerated from the seed on the
test side (see make_golden.py).
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


def main():
    torch.manual_seed(0)
    cfg, wseed, iseed, t = config.SD21_UNET, 31, 32, 981.0
    sd = config.random_state_dict(config.unet_param_shapes(cfg), seed=wseed)
    x, c = unet_inputs(cfg, iseed)
    m = ref_unet.build_unet(cfg, sd, impl="ORIGINAL")
    with torch.no_grad():
        y = m(x, torch.tensor([t, t]), c)[0].numpy()
    np.savez_compressed(os.path.join(OUT, "unet_sd21_768.npz"), weight_seed=wseed, input_seed=iseed, timestep=t,
                        fingerprint=fingerprint(sd), noise_pred_ORIGINAL=y.astype(np.float32))
    print("sd21_768", y.shape, float(np.abs(y).max()))


if __name__ == "__main__":
    main()
