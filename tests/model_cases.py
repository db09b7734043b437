"""The shipped models the per-launch replays run (test_gemm_plans_gpu.py: GEMM / convolution launches,
test_op_launches_gpu.py: every other kernel): random-init weights at the shapes the pipelines use, and random inputs of
each model's declared input spec.  Both replays run every name of SHIPPED."""
import torch

# name -> the pipeline path that launches that model at that shape
SHIPPED_PATHS = {
    "sd21_b2": "SD-2.1-base txt2img at 512^2, one image per call (UNet batch 2 under CFG)",
    "sd21_b16": "SD-2.1-base at 512^2, 8 images per call: the benchmark's batch",
    "sd15_b2": "SD 1.4 / 1.5 txt2img at 512^2 (head dims 40 / 80 / 160, 768-wide text states)",
    "sd21_768_b2": "SD 2.0 / 2.1 768-v txt2img at 768^2 (96^2 latents)",
    "sdxl_768_b2": "SDXL-base at 768^2 (96^2 latents)",
    "sdxl_1024_b2": "SDXL-base at its default 1024^2 (from_pretrained with no size: sample_size 128)",
    "sdxl_refiner_1024_b2": "SDXL refiner (from_pretrained(refiner_dir=...)) at 1024^2",
    "sdxl_refiner_768_b2": "SDXL refiner at 768^2",
    "controlnet_sd21": "ControlNet with SD-2.1-base at 512^2",
    "controlnet_sd15": "ControlNet with SD 1.5 (config.SD15_CONTROLNET) at 512^2",
    "controlnet_sd21_768": "ControlNet with SD-2.1 768-v at 768^2",
    "vae_decoder": "SD 1.x / 2.x VAE decode in fp16, 64^2 latents -> 512^2",
    "vae_decoder_768": "SD-2.1 768-v VAE decode in fp16, 96^2 latents -> 768^2",
    "vae_decoder_bf16": "SDXL VAE decode (force_upcast: bf16), 128^2 latents -> 1024^2",
    "vae_decoder_bf16_768": "SDXL VAE decode in bf16 at 768^2 (96^2 latents)",
    "vae_encoder_512": "SD 1.x / 2.x img2img / inpainting encode in fp16 at 512^2",
    "vae_encoder_768": "SD-2.1 768-v img2img / inpainting encode in fp16 at 768^2",
    "vae_encoder_bf16": "SDXL img2img encode in bf16 at 512^2",
    "vae_encoder_bf16_1024": "SDXL img2img encode in bf16 at 1024^2",
    "openclip_h": "SD-2.x text encoder (OpenCLIP ViT-H/14, penultimate layer)",
    "clip_l": "SD-1.x text encoder (CLIP ViT-L/14) and SDXL's first encoder",
    "openclip_bigg": "SDXL's second text encoder and the refiner's only one (OpenCLIP ViT-bigG/14)",
}
SHIPPED = list(SHIPPED_PATHS)


def model_inputs(m, seed):
    """Random inputs of a model's declared input spec (timesteps mid-schedule, token ids of a short prompt).  SDXL time
    ids hold the model's image size: six (original size, crop, target size) for the base, five (original size, crop,
    aesthetic score 6) for the refiner."""
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
            h, w = 8.0 * m.h, 8.0 * m.w
            ids = {6: [h, w, 0.0, 0.0, h, w], 5: [h, w, 0.0, 0.0, 6.0]}[shp[1]]
            v = torch.tensor(ids).expand(shp).contiguous()
        elif k == "controlnet_cond":
            v = torch.rand(shp, generator=g)
        else:
            v = torch.randn(shp, generator=g)
        kw[k] = v.numpy().astype(np.dtype(spec["dtype"]))
    return kw


def _latent_hw(name, default):
    return 128 if "1024" in name else (96 if "768" in name else default)


def build(name):
    """The model of a SHIPPED name.  UNets (sd21_*, sd21_768_*, sd15_*, sdxl_*, sdxl_refiner_*): batch 16 with "b16"
    in the name, else 2; 64^2 latents for SD 1.x / 2.x-base, 96^2 for 768-v and "768", 128^2 for "1024".  ControlNets
    at batch 2.  VAEs at batch 1: decoders take latents (64^2, or 128^2 for the bf16 one, unless the name says 768),
    encoders images (512^2 unless the name says 768 / 1024); "bf16" runs the SDXL VAE's bf16 engine, else the SD VAE in
    fp16.  The text encoders openclip_h, clip_l and openclip_bigg at batch 2."""
    from b200sd import config as C

    if name.startswith(("sd21", "sd15", "sdxl")):
        from b200sd.model import UNetModel
        v768 = name.startswith("sd21_768")
        if name.startswith("sdxl_refiner"):
            cfg = C.SDXL_REFINER_UNET
        else:
            cfg = C.SD21_UNET if v768 else {"sd21": C.SD21_BASE_UNET, "sd15": C.SD15_UNET, "sdxl": C.SDXL_BASE_UNET}[name[:4]]
        batch = 16 if "b16" in name else 2
        hw = _latent_hw(name, 96 if (name.startswith("sdxl") or v768) else 64)
        sd = C.random_state_dict(C.unet_param_shapes(cfg), seed=5, dtype=torch.float16)
        return UNetModel(cfg, sd, batch=batch, height=hw, width=hw, use_cuda_graph=False)
    if name.startswith("controlnet"):
        from b200sd.controlnet import ControlNetModel
        cfg = C.SD15_CONTROLNET if name.startswith("controlnet_sd15") else C.SD21_CONTROLNET
        sd = C.random_state_dict(C.controlnet_param_shapes(cfg), seed=6, dtype=torch.float16)
        hw = _latent_hw(name, 64)
        return ControlNetModel(cfg, sd, batch=2, height=hw, width=hw, use_cuda_graph=False)
    if name.startswith("vae_decoder"):
        from b200sd.vae import VAEDecoderModel
        bf16 = "bf16" in name
        vcfg = C.SDXL_VAE if bf16 else C.SD_VAE
        sd = C.random_state_dict(C.vae_decoder_param_shapes(vcfg), seed=7, dtype=torch.float16)
        hw = _latent_hw(name, 128 if bf16 else 64)
        return VAEDecoderModel(vcfg, sd, batch=1, height=hw, width=hw, dtype=torch.bfloat16 if bf16 else torch.float16)
    if name.startswith("vae_encoder"):
        from b200sd.vae import VAEEncoderModel
        bf16 = "bf16" in name
        vcfg = C.SDXL_VAE if bf16 else C.SD_VAE
        sd = C.random_state_dict(C.vae_encoder_param_shapes(vcfg), seed=10, dtype=torch.float16)
        px = 8 * _latent_hw(name, 64)
        return VAEEncoderModel(vcfg, sd, batch=1, height=px, width=px, dtype=torch.bfloat16 if bf16 else torch.float16)
    from b200sd.text_encoder import TextEncoderModel
    cfg = {"openclip_h": C.OPENCLIP_H_TEXT, "clip_l": C.CLIP_L_TEXT, "openclip_bigg": C.OPENCLIP_BIGG_TEXT}[name]
    return TextEncoderModel(cfg, C.random_clip_text_state_dict(cfg, seed=8, dtype=torch.float16), batch=2)
