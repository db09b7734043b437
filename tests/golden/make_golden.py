"""Generates the golden fixtures under tests/golden/ by running the UNMODIFIED reference modules
(python_coreml_stable_diffusion.{unet,attention,layer_norm}) imported from /root/reference through
oracle/ref_unet.py.  Run in the build container only (the GPU box has no reference tree):

    python tests/golden/make_golden.py

Weights are not stored: they are regenerated from a seed by b200sd.config.random_state_dict (CPU
torch generator, deterministic for a given torch build); a fingerprint of them is stored so a
generator mismatch is detected instead of silently failing parity.
"""
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)

from b200sd import config  # noqa: E402
from oracle import ref_unet  # noqa: E402

OUT = os.path.dirname(os.path.abspath(__file__))


def fingerprint(sd):
    keys = sorted(sd.keys())
    picks = [keys[0], keys[len(keys) // 2], keys[-1]]
    return np.array([float(sd[k].double().sum()) for k in picks] + [float(len(keys))])


def unet_inputs(cfg, seed, batch=2, seq=77, size=None):
    g = torch.Generator().manual_seed(seed)
    s = size or cfg["sample_size"]
    x = torch.randn(batch, cfg["in_channels"], s, s, generator=g)
    c = torch.randn(batch, cfg["cross_attention_dim"], 1, seq, generator=g)
    return x, c


def main():
    torch.manual_seed(0)
    ref = ref_unet.load()
    # ---- full UNet, three attention implementations, tiny + SD-2.1-base -----------------------
    for name, cfg, wseed, iseed, t in [("tiny", config.TINY_UNET, 1, 2, 981.0),
                                       ("sd21", config.SD21_BASE_UNET, 1, 2, 981.0)]:
        sd = config.random_state_dict(config.unet_param_shapes(cfg), seed=wseed)
        x, c = unet_inputs(cfg, iseed)
        ts = torch.tensor([t, t])
        outs = {}
        for impl in ("ORIGINAL", "SPLIT_EINSUM", "SPLIT_EINSUM_V2"):
            if name == "sd21" and impl != "ORIGINAL":
                continue
            m = ref_unet.build_unet(cfg, sd, impl=impl)
            with torch.no_grad():
                outs[impl] = m(x, ts, c)[0].numpy()
        np.savez_compressed(os.path.join(OUT, f"unet_{name}.npz"), weight_seed=wseed, input_seed=iseed,
                            timestep=t, fingerprint=fingerprint(sd),
                            **{f"noise_pred_{k}": v.astype(np.float32) for k, v in outs.items()})
        print(name, {k: float(np.abs(v).max()) for k, v in outs.items()})

    # ---- SDXL-style UNet (UNet2DConditionModelXL) and ControlNetModel, tiny configs ------------------------
    cfg = config.TINY_XL_UNET
    sd = config.random_state_dict(config.unet_param_shapes(cfg), seed=3)
    x, c = unet_inputs(cfg, 9)
    gg = torch.Generator().manual_seed(10)
    tid = torch.tensor([[64.0, 64.0, 0.0, 0.0, 64.0, 64.0]] * 2)
    te = torch.randn(2, 64, generator=gg)
    m = ref_unet.build_unet(cfg, sd, xl=True, impl="SPLIT_EINSUM")
    with torch.no_grad():
        y = m(x, torch.tensor([981.0, 981.0]), c, tid, te)[0].numpy()
    np.savez_compressed(os.path.join(OUT, "unet_tiny_xl.npz"), weight_seed=3, input_seed=9, fingerprint=fingerprint(sd),
                        text_embeds=te.numpy(), time_ids=tid.numpy(), noise_pred=y.astype(np.float32))
    ccfg = config.TINY_CONTROLNET
    csd = config.random_state_dict(config.controlnet_param_shapes(ccfg), seed=4)
    x, c = unet_inputs(config.TINY_UNET, 6)
    cond = torch.rand(2, 3, 128, 128, generator=torch.Generator().manual_seed(7))
    cn = ref_unet.build_controlnet(ccfg, csd)
    with torch.no_grad():
        down, mid = cn(x.clone(), torch.tensor([501.0, 501.0]), c, cond)
    np.savez_compressed(os.path.join(OUT, "controlnet_tiny.npz"), weight_seed=4, input_seed=6, cond_seed=7,
                        fingerprint=fingerprint(csd),
                        **{f"residual_{i}": r.numpy().astype(np.float32) for i, r in enumerate(list(down) + [mid])})
    print("xl + controlnet done")

    # ---- attention variants + LayerNormANE on their own ---------------------------------------
    g = torch.Generator().manual_seed(5)
    q = torch.randn(2, 128, 1, 200, generator=g)
    k = torch.randn(2, 128, 1, 77, generator=g)
    v = torch.randn(2, 128, 1, 77, generator=g)
    mask = torch.zeros(2, 77, 1, 1)
    mask[:, 50:] = -1e4
    att = {}
    for nm, fn in (("original", ref.attention.original), ("split_einsum", ref.attention.split_einsum),
                   ("split_einsum_v2", ref.attention.split_einsum_v2)):
        att[nm] = fn(q.clone(), k.clone(), v.clone(), None, 2, 64).numpy()
    att["split_einsum_masked"] = ref.attention.split_einsum(q.clone(), k.clone(), v.clone(), mask, 2, 64).numpy()
    ln = ref.layer_norm.LayerNormANE(128)
    with torch.no_grad():
        ln.weight.copy_(torch.randn(128, generator=g))
        ln.bias.copy_(torch.randn(128, generator=g))
        ln_out = ln(q.clone()).numpy()
    temb = ref.unet.get_timestep_embedding(torch.tensor([981.0, 1.0, 500.0]), 320, flip_sin_to_cos=True,
                                           downscale_freq_shift=0).numpy()
    s = 4  # outputs are kept at every 4th query position (keeps the fixture under 1 MB)
    np.savez_compressed(os.path.join(OUT, "blocks.npz"), q=q.numpy(), k=k.numpy(), v=v.numpy(), mask=mask.numpy(),
                        ln_weight=ln.weight.detach().numpy(), ln_bias=ln.bias.detach().numpy(), ln_out=ln_out[..., ::s],
                        temb=temb, out_stride=s, **{f"attn_{k_}": v_[..., ::s] for k_, v_ in att.items()})
    print("blocks done")


if __name__ == "__main__":
    main()
