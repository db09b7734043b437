"""The shipped models the per-launch replays run (test_gemm_plans_gpu.py: GEMM / convolution launches,
test_op_launches_gpu.py: every other kernel): random-init weights at the shapes the pipelines use, and random inputs of
each model's declared input spec.  Both replays run every name of SHIPPED.  A name may carry its image size in pixels,
`<height>x<width>` (latent_hw): the non-square sizes are where a kernel or the host could confuse h with w unseen."""
import re

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
    "sd15_512x768_b2": "SD 1.x txt2img at 512x768 (portrait): 64x96 latents down to 8x12, mid-block attention over 96",
    "sd15_768x512_b2": "SD 1.x txt2img at 768x512 (landscape): 96x64 latents down to 12x8",
    "sd21_576x576_b2": "SD-2.1-base txt2img at 576^2: 72^2 latents, stride 2 from 18^2 to an odd 9^2 (81 tokens)",
    "sdxl_768x1344_b2": "SDXL-base on its 768x1344 aspect-ratio bucket: attention over 4032 and 1008 tokens",
    "sdxl_1216x832_b2": "SDXL-base on its 1216x832 bucket: attention over 3952 and 988 tokens",
    "sdxl_refiner_768x1344_b2": "SDXL refiner at 768x1344: a 12x21 deepest map, mid-block attention over 252 tokens",
    "controlnet_sd21": "ControlNet with SD-2.1-base at 512^2",
    "controlnet_sd15": "ControlNet with SD 1.5 (config.SD15_CONTROLNET) at 512^2",
    "controlnet_sd21_768": "ControlNet with SD-2.1 768-v at 768^2",
    "controlnet_sd15_512x768": "ControlNet with SD 1.5 at 512x768: the hint encoder's stride-2 chain on that image",
    "vae_decoder": "SD 1.x / 2.x VAE decode in fp16, 64^2 latents -> 512^2",
    "vae_decoder_768": "SD-2.1 768-v VAE decode in fp16, 96^2 latents -> 768^2",
    "vae_decoder_bf16": "SDXL VAE decode (force_upcast: bf16), 128^2 latents -> 1024^2",
    "vae_decoder_bf16_768": "SDXL VAE decode in bf16 at 768^2 (96^2 latents)",
    "vae_decoder_512x768": "SD 1.x VAE decode in fp16 at 512x768: mid-block softmax over 6144 columns",
    "vae_decoder_bf16_768x1344": "SDXL VAE decode in bf16 at 768x1344: mid-block softmax over 16128 columns",
    "vae_encoder_512": "SD 1.x / 2.x img2img / inpainting encode in fp16 at 512^2",
    "vae_encoder_768": "SD-2.1 768-v img2img / inpainting encode in fp16 at 768^2",
    "vae_encoder_bf16": "SDXL img2img encode in bf16 at 512^2",
    "vae_encoder_bf16_1024": "SDXL img2img encode in bf16 at 1024^2",
    "vae_encoder_768x512": "SD 1.x img2img encode in fp16 at 768x512: stride-2 convolutions padded after only",
    "vae_encoder_bf16_1216x832": "SDXL img2img encode in bf16 at 1216x832",
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


def latent_hw(name):
    """(height, width) of the latents of a SHIPPED UNet, ControlNet or VAE name (a VAE encoder's image is 8 times as
    large): the explicit pixel size `<height>x<width>` when the name has one, else square: 128^2 with "1024" in the
    name, 96^2 with "768", otherwise the family's default (96^2 for SDXL-base, the refiner and SD-2.1 768-v, 128^2 for
    the bf16 VAE decoder, 64^2 for the rest)."""
    m = re.search(r"_(\d+)x(\d+)(?:_|$)", name)
    if m:
        h, w = int(m.group(1)), int(m.group(2))
        assert h % 8 == 0 and w % 8 == 0, name
        return h // 8, w // 8
    if "1024" in name:
        return 128, 128
    if "768" in name or name.startswith("sdxl"):
        return 96, 96
    return (128, 128) if name.startswith("vae_decoder_bf16") else (64, 64)


def build(name):
    """The model of a SHIPPED name.  UNets (sd21_*, sd21_768_*, sd15_*, sdxl_*, sdxl_refiner_*): batch 16 with "b16"
    in the name, else 2.  ControlNets at batch 2.  VAEs at batch 1: decoders take latents, encoders images; "bf16" runs
    the SDXL VAE's bf16 engine, else the SD VAE in fp16.  Sizes from latent_hw.  The text encoders openclip_h, clip_l
    and openclip_bigg at batch 2."""
    from b200sd import config as C

    if name.startswith(("sd21", "sd15", "sdxl")):
        from b200sd.model import UNetModel
        v768 = name.startswith("sd21_768")
        if name.startswith("sdxl_refiner"):
            cfg = C.SDXL_REFINER_UNET
        else:
            cfg = C.SD21_UNET if v768 else {"sd21": C.SD21_BASE_UNET, "sd15": C.SD15_UNET, "sdxl": C.SDXL_BASE_UNET}[name[:4]]
        batch = 16 if "b16" in name else 2
        h, w = latent_hw(name)
        sd = C.random_state_dict(C.unet_param_shapes(cfg), seed=5, dtype=torch.float16)
        return UNetModel(cfg, sd, batch=batch, height=h, width=w, use_cuda_graph=False)
    if name.startswith("controlnet"):
        from b200sd.controlnet import ControlNetModel
        cfg = C.SD15_CONTROLNET if name.startswith("controlnet_sd15") else C.SD21_CONTROLNET
        sd = C.random_state_dict(C.controlnet_param_shapes(cfg), seed=6, dtype=torch.float16)
        h, w = latent_hw(name)
        return ControlNetModel(cfg, sd, batch=2, height=h, width=w, use_cuda_graph=False)
    if name.startswith("vae_decoder"):
        from b200sd.vae import VAEDecoderModel
        bf16 = "bf16" in name
        vcfg = C.SDXL_VAE if bf16 else C.SD_VAE
        sd = C.random_state_dict(C.vae_decoder_param_shapes(vcfg), seed=7, dtype=torch.float16)
        h, w = latent_hw(name)
        return VAEDecoderModel(vcfg, sd, batch=1, height=h, width=w, dtype=torch.bfloat16 if bf16 else torch.float16)
    if name.startswith("vae_encoder"):
        from b200sd.vae import VAEEncoderModel
        bf16 = "bf16" in name
        vcfg = C.SDXL_VAE if bf16 else C.SD_VAE
        sd = C.random_state_dict(C.vae_encoder_param_shapes(vcfg), seed=10, dtype=torch.float16)
        h, w = latent_hw(name)
        return VAEEncoderModel(vcfg, sd, batch=1, height=8 * h, width=8 * w,
                               dtype=torch.bfloat16 if bf16 else torch.float16)
    from b200sd.text_encoder import TextEncoderModel
    cfg = {"openclip_h": C.OPENCLIP_H_TEXT, "clip_l": C.CLIP_L_TEXT, "openclip_bigg": C.OPENCLIP_BIGG_TEXT}[name]
    return TextEncoderModel(cfg, C.random_clip_text_state_dict(cfg, seed=8, dtype=torch.float16), batch=2)
