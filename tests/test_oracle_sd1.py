"""CPU tests that pin the oracle (oracle/restated.py) and the SD-1 configs to the golden vectors of the unmodified
reference modules for Stable Diffusion 1.x (tests/golden/make_golden_sd1.py): 8 heads per block, head dims 40 / 80 / 160."""
import math
import os

import numpy as np
import pytest
import torch

from b200sd import config
from oracle import restated as R

GOLD = os.path.join(os.path.dirname(__file__), "golden")


def _fingerprint(sd):
    keys = sorted(sd.keys())
    picks = [keys[0], keys[len(keys) // 2], keys[-1]]
    return np.array([float(sd[k].double().sum()) for k in picks] + [float(len(keys))])


def _inputs(cfg, seed, batch=2, seq=77):
    g = torch.Generator().manual_seed(seed)
    s = cfg["sample_size"]
    return (torch.randn(batch, cfg["in_channels"], s, s, generator=g),
            torch.randn(batch, cfg["cross_attention_dim"], 1, seq, generator=g))


def test_sd1_configs():
    """SD-1.5 is SD-2.1-base with 8 heads and 768-wide text states: the published 859,520,964-parameter UNet."""
    n = sum(math.prod(s) for s in config.unet_param_shapes(config.SD15_UNET).values())
    assert n == 859_520_964
    for cfg in (config.SD15_UNET, config.TINY_SD1_UNET, config.SD15_CONTROLNET, config.TINY_SD1_CONTROLNET):
        heads = config._as_list(cfg["attention_head_dim"], len(cfg["block_out_channels"]))
        assert {c // h for c, h in zip(cfg["block_out_channels"], heads)} <= {40, 80, 160}
    heads = config.TINY_SD1_UNET["attention_head_dim"]
    assert [c // h for c, h in zip(config.TINY_SD1_UNET["block_out_channels"], heads)] == [40, 80, 160]


@pytest.mark.parametrize("name,cfg", [("tiny_sd1", config.TINY_SD1_UNET), ("sd15", config.SD15_UNET)])
def test_restated_sd1_unet_matches_reference_golden(name, cfg):
    gold = np.load(os.path.join(GOLD, f"unet_{name}.npz"))
    sd = config.random_state_dict(config.unet_param_shapes(cfg), seed=int(gold["weight_seed"]))
    assert np.allclose(_fingerprint(sd), gold["fingerprint"], rtol=1e-6), "weight generator drifted"
    x, c = _inputs(cfg, int(gold["input_seed"]))
    t = torch.tensor([float(gold["timestep"])] * 2)
    with torch.no_grad():
        y = R.unet_forward(sd, cfg, x, t, c).numpy()
    keys = [k for k in gold.files if k.startswith("noise_pred_")]
    assert keys
    for key in keys:
        assert np.abs(y - gold[key]).max() < 2e-5, key
        assert R.compute_psnr(torch.from_numpy(y), torch.from_numpy(gold[key])) > 100


def test_restated_sd1_controlnet_matches_reference_golden():
    gold = np.load(os.path.join(GOLD, "controlnet_tiny_sd1.npz"))
    cfg = config.TINY_SD1_CONTROLNET
    sd = config.random_state_dict(config.controlnet_param_shapes(cfg), seed=int(gold["weight_seed"]))
    assert np.allclose(_fingerprint(sd), gold["fingerprint"], rtol=1e-6)
    x, c = _inputs(config.TINY_SD1_UNET, int(gold["input_seed"]))
    cond = torch.rand(2, 3, 128, 128, generator=torch.Generator().manual_seed(int(gold["cond_seed"])))
    st = int(gold["stride"])
    with torch.no_grad():
        outs = R.controlnet_forward(sd, cfg, x, torch.tensor([501.0, 501.0]), c, cond.half().float())
    assert len(outs) == 7
    for i, o in enumerate(outs):
        ref = torch.from_numpy(gold[f"residual_{i}"].astype(np.float32))
        err = float((o[:, :, ::st, ::st] - ref).abs().max())
        assert err < 2e-3 * max(1.0, float(ref.abs().max())), (i, err)  # the fixture is stored in fp16
