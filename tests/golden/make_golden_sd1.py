"""Golden fixtures for Stable Diffusion 1.x (8 heads per block: head dims 40, 80 and 160), produced by the UNMODIFIED
reference modules (python_coreml_stable_diffusion.{unet,controlnet}) through oracle/ref_unet.py on the CPU in fp32.
Build container only:

    python tests/golden/make_golden_sd1.py

Writes
  unet_tiny_sd1.npz        config.TINY_SD1_UNET, all three attention implementations
  unet_sd15.npz            config.SD15_UNET (859.5 M parameters), 64x64 latents, ORIGINAL
  controlnet_tiny_sd1.npz  config.TINY_SD1_CONTROLNET residuals, fp16, sub-sampled [:, :, ::stride, ::stride]
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
CN_STRIDE = 2


def main():
    torch.manual_seed(0)
    for name, cfg, wseed, iseed, t, impls in [
            ("tiny_sd1", config.TINY_SD1_UNET, 21, 22, 981.0, ("ORIGINAL", "SPLIT_EINSUM", "SPLIT_EINSUM_V2")),
            ("sd15", config.SD15_UNET, 23, 24, 981.0, ("ORIGINAL",))]:
        sd = config.random_state_dict(config.unet_param_shapes(cfg), seed=wseed)
        x, c = unet_inputs(cfg, iseed)
        ts = torch.tensor([t, t])
        outs = {}
        for impl in impls:
            m = ref_unet.build_unet(cfg, sd, impl=impl)
            with torch.no_grad():
                outs[impl] = m(x, ts, c)[0].numpy()
            del m
        np.savez_compressed(os.path.join(OUT, f"unet_{name}.npz"), weight_seed=wseed, input_seed=iseed,
                            timestep=t, fingerprint=fingerprint(sd),
                            **{f"noise_pred_{k}": v.astype(np.float32) for k, v in outs.items()})
        print(name, {k: float(np.abs(v).max()) for k, v in outs.items()})

    ccfg = config.TINY_SD1_CONTROLNET
    csd = config.random_state_dict(config.controlnet_param_shapes(ccfg), seed=25)
    x, c = unet_inputs(config.TINY_SD1_UNET, 26)
    cond = torch.rand(2, 3, 128, 128, generator=torch.Generator().manual_seed(27))
    cn = ref_unet.build_controlnet(ccfg, csd)
    with torch.no_grad():
        down, mid = cn(x.clone(), torch.tensor([501.0, 501.0]), c, cond.half().float())
    res = list(down) + [mid]
    print([tuple(r.shape) for r in res], [round(float(r.abs().max()), 3) for r in res])
    np.savez_compressed(os.path.join(OUT, "controlnet_tiny_sd1.npz"), weight_seed=25, input_seed=26, cond_seed=27,
                        stride=CN_STRIDE, fingerprint=fingerprint(csd),
                        **{f"residual_{i}": r[:, :, ::CN_STRIDE, ::CN_STRIDE].numpy().astype(np.float16)
                           for i, r in enumerate(res)})


if __name__ == "__main__":
    main()
