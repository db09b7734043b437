"""The shipped models the per-launch replays run (test_gemm_plans_gpu.py: GEMM / convolution launches,
test_op_launches_gpu.py: every other kernel): random-init weights at the shapes the pipelines use, and random inputs of
each model's declared input spec."""
import torch


def model_inputs(m, seed):
    """Random inputs of a model's declared input spec (timesteps mid-schedule, token ids of a short prompt)."""
    import numpy as np

    g = torch.Generator().manual_seed(seed)
    kw = {}
    for k, spec in m.expected_inputs.items():
        shp = tuple(spec["shape"])
        if k == "timestep":
            v = torch.full(shp, 501.0)
        elif k == "input_ids":
            v = torch.randint(0, 49406, shp, generator=g).float()
            v[:, 0], v[:, 20:] = 49406, 49407
        elif k == "time_ids":
            v = torch.tensor([768.0, 768.0, 0.0, 0.0, 768.0, 768.0])[: shp[1]].expand(shp).contiguous()
        elif k == "controlnet_cond":
            v = torch.rand(shp, generator=g)
        else:
            v = torch.randn(shp, generator=g)
        kw[k] = v.numpy().astype(np.dtype(spec["dtype"]))
    return kw


def build(name):
    """sd21_* (SD-2.1-base, 64^2 latents), sd21_768_* (SD-2.1 768-v, 96^2 latents), sd15_*, sdxl_* (96^2 latents), with
    "b16" in the name at batch 16, else 2; controlnet_sd21; vae_decoder (fp16, 64 -> 512); vae_decoder_bf16 (the SDXL
    VAE's bf16 engine, 128 -> 1024); vae_encoder_bf16 (bf16, 512 -> 64); the text encoders openclip_h, clip_l and
    openclip_bigg."""
    from b200sd import config as C

    if name.startswith(("sd21", "sd15", "sdxl")):
        from b200sd.model import UNetModel
        v768 = name.startswith("sd21_768")
        cfg = C.SD21_UNET if v768 else {"sd21": C.SD21_BASE_UNET, "sd15": C.SD15_UNET, "sdxl": C.SDXL_BASE_UNET}[name[:4]]
        batch = 16 if "b16" in name else 2
        hw = 96 if (name.startswith("sdxl") or v768) else 64
        sd = C.random_state_dict(C.unet_param_shapes(cfg), seed=5, dtype=torch.float16)
        return UNetModel(cfg, sd, batch=batch, height=hw, width=hw, use_cuda_graph=False)
    if name == "controlnet_sd21":
        from b200sd.controlnet import ControlNetModel
        cfg = C.SD21_CONTROLNET
        sd = C.random_state_dict(C.controlnet_param_shapes(cfg), seed=6, dtype=torch.float16)
        return ControlNetModel(cfg, sd, batch=2, height=64, width=64, use_cuda_graph=False)
    if name == "vae_decoder":
        from b200sd.vae import VAEDecoderModel
        sd = C.random_state_dict(C.vae_decoder_param_shapes(C.SD_VAE), seed=7, dtype=torch.float16)
        return VAEDecoderModel(C.SD_VAE, sd, batch=1, height=64, width=64)
    if name == "vae_decoder_bf16":
        from b200sd.vae import VAEDecoderModel
        sd = C.random_state_dict(C.vae_decoder_param_shapes(C.SDXL_VAE), seed=7, dtype=torch.float16)
        return VAEDecoderModel(C.SDXL_VAE, sd, batch=1, height=128, width=128, dtype=torch.bfloat16)
    if name == "vae_encoder_bf16":
        from b200sd.vae import VAEEncoderModel
        sd = C.random_state_dict(C.vae_encoder_param_shapes(C.SDXL_VAE), seed=10, dtype=torch.float16)
        return VAEEncoderModel(C.SDXL_VAE, sd, batch=1, height=512, width=512, dtype=torch.bfloat16)
    from b200sd.text_encoder import TextEncoderModel
    cfg = {"openclip_h": C.OPENCLIP_H_TEXT, "clip_l": C.CLIP_L_TEXT, "openclip_bigg": C.OPENCLIP_BIGG_TEXT}[name]
    return TextEncoderModel(cfg, C.random_clip_text_state_dict(cfg, seed=8, dtype=torch.float16), batch=2)
