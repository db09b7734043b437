"""Weight ingestion from diffusers-layout checkpoints (SURVEY 8f N4, host side).

The reference builds its networks from the diffusers pipeline's modules and loads their ``state_dict()`` unchanged
(``torch2coreml.py:915-918``: ``reference_unet.load_state_dict(pipe.unet.state_dict())``; the pre-hooks of
``unet.py:121-138`` only reshape ``nn.Linear`` weights to 1x1 convolutions).  The engines of this package take those
same parameter names, so ingestion is: read ``<model dir>/<component>/diffusion_pytorch_model.safetensors`` (or a
sharded / ``.bin`` variant), check it against the architecture schema, hand it to the engine.
"""
from __future__ import annotations

import json
import os

import torch

from . import config as C

_SCHEMAS = {
    "unet": C.unet_param_shapes,
    "controlnet": C.controlnet_param_shapes,
    "vae_decoder": C.vae_decoder_param_shapes,
    "vae_encoder": C.vae_encoder_param_shapes,
    "text_encoder": C.clip_text_param_shapes,
    "safety_checker": C.safety_checker_param_shapes,
}
# AutoencoderKL checkpoints written before diffusers 0.18 name the mid-block attention projections query / key / value /
# proj_attn (diffusers remaps them when it loads the file); the engines use the current names
_VAE_ATTN_RENAMES = {".query.": ".to_q.", ".key.": ".to_k.", ".value.": ".to_v.", ".proj_attn.": ".to_out.0."}
_FILES = ("diffusion_pytorch_model.safetensors", "model.safetensors", "diffusion_pytorch_model.fp16.safetensors",
          "model.fp16.safetensors", "diffusion_pytorch_model.bin", "pytorch_model.bin")


def read_state_dict(path: str) -> dict:
    """A .safetensors / .bin file, a sharded ``*.index.json``, or a component directory holding one of them."""
    if os.path.isdir(path):
        for f in _FILES:
            if os.path.exists(os.path.join(path, f)):
                return read_state_dict(os.path.join(path, f))
        idx = [f for f in os.listdir(path) if f.endswith(".index.json")]
        if idx:
            return read_state_dict(os.path.join(path, idx[0]))
        raise FileNotFoundError(f"no checkpoint file found under {path}")
    if path.endswith(".index.json"):
        with open(path) as f:
            shards = sorted(set(json.load(f)["weight_map"].values()))
        sd = {}
        for s in shards:
            sd.update(read_state_dict(os.path.join(os.path.dirname(path), s)))
        return sd
    if path.endswith(".safetensors"):
        from safetensors.torch import load_file
        return load_file(path, device="cpu")
    return torch.load(path, map_location="cpu", weights_only=True)


def _canonical(shape):
    """Linear weights may be stored as [out, in] (diffusers) or [out, in, 1, 1] (after the reference's pre-hooks)."""
    shape = tuple(shape)
    return shape[:2] if len(shape) == 4 and shape[2:] == (1, 1) else shape


def remap_legacy_vae_keys(sd: dict) -> dict:
    """Deprecated AutoencoderKL attention names -> current ones (values untouched; [C, C, 1, 1] vs [C, C] is accepted
    by the shape check below)."""
    out = {}
    for k, v in sd.items():
        if ".attentions." in k:
            for old, new in _VAE_ATTN_RENAMES.items():
                if old in k:
                    k = k.replace(old, new)
                    break
        out[k] = v
    return out


def check_state_dict(component: str, cfg: dict, sd: dict, allow_extra=True) -> dict:
    """Validates names and shapes against the architecture schema; returns the subset the engine consumes.
    ``vae_decoder`` / ``vae_encoder`` accept a full AutoencoderKL state dict (the other half is dropped)."""
    want = _SCHEMAS[component](cfg)
    if component.startswith("vae"):
        sd = remap_legacy_vae_keys(sd)
    missing = [k for k in want if k not in sd]
    if missing:
        raise KeyError(f"{component}: {len(missing)} parameters missing from the checkpoint, e.g. {missing[:3]}")
    bad = [(k, tuple(sd[k].shape), tuple(want[k])) for k in want if _canonical(sd[k].shape) != _canonical(want[k])]
    if bad:
        raise ValueError(f"{component}: shape mismatch for {len(bad)} parameters, e.g. {bad[:3]}")
    extra = [k for k in sd if k not in want]
    if extra and not allow_extra:
        raise KeyError(f"{component}: unexpected parameters, e.g. {extra[:3]}")
    return {k: sd[k] for k in want}


def load_component(model_dir: str, component: str, cfg: dict) -> dict:
    """``model_dir`` is a diffusers pipeline directory (``unet/``, ``vae/``, ``text_encoder/``, ...)."""
    sub = {"unet": "unet", "controlnet": "", "vae_decoder": "vae", "vae_encoder": "vae", "text_encoder": "text_encoder",
           "text_encoder_2": "text_encoder_2", "unet_refiner": "unet"}.get(component, component)
    schema = "text_encoder" if component == "text_encoder_2" else ("unet" if component == "unet_refiner" else component)
    return check_state_dict(schema, cfg, read_state_dict(os.path.join(model_dir, sub) if sub else model_dir))


def read_config(model_dir: str, component: str) -> dict:
    """``<model_dir>/<component>/config.json`` (scheduler: ``scheduler_config.json``) of a diffusers pipeline directory,
    reduced to the keys the engines read (private ``_class_name`` / ``_diffusers_version`` entries dropped)."""
    name = "scheduler_config.json" if component == "scheduler" else "config.json"
    with open(os.path.join(model_dir, component, name)) as f:
        cfg = json.load(f)
    return {k: (tuple(v) if isinstance(v, list) else v) for k, v in cfg.items() if not k.startswith("_")}


# CLIPImageProcessor's defaults (transformers 4.44.2, the release the reference pins)
OPENAI_CLIP_MEAN = (0.48145466, 0.4578275, 0.40821073)
OPENAI_CLIP_STD = (0.26862954, 0.26130258, 0.27577711)
PREPROCESS_DEFAULTS = dict(size=224, crop_h=224, crop_w=224, mean=OPENAI_CLIP_MEAN, std=OPENAI_CLIP_STD)


def _edge(raw, key, default):
    """``size`` / ``crop_size``: an int, or a dict (``shortest_edge`` for size; ``height`` / ``width`` for crop_size)."""
    v = raw.get(key, default)
    if isinstance(v, bool) or not isinstance(v, (int, dict)):
        raise ValueError(f"preprocessor_config.json: {key}={v!r} is neither an int nor a dict")
    return v


def preprocessor_config(raw: dict) -> dict:
    """A ``feature_extractor/preprocessor_config.json`` (CLIPFeatureExtractor / CLIPImageProcessor) -> dict(size,
    crop_h, crop_w, mean, std).  Only the pipeline the safety checker was trained with runs on the device: BICUBIC
    (resample = 3) resize of the shortest edge, centre crop, rescale by 1/255 and normalise.  Anything else raises a
    ValueError that names the key."""
    for key in ("do_resize", "do_center_crop", "do_rescale", "do_normalize"):
        if raw.get(key, True) is not True:
            raise ValueError(f"preprocessor_config.json: {key}={raw[key]!r}; the safety checker's preprocessing "
                             "needs resize, centre crop, rescale and normalise")
    if raw.get("resample", 3) != 3:
        raise ValueError(f"preprocessor_config.json: resample={raw['resample']!r}; only 3 (BICUBIC) is implemented")
    if abs(float(raw.get("rescale_factor", 1 / 255)) - 1 / 255) > 1e-12:
        raise ValueError(f"preprocessor_config.json: rescale_factor={raw['rescale_factor']!r}; only 1/255 is "
                         "implemented")
    size = _edge(raw, "size", 224)
    if isinstance(size, dict):
        if "shortest_edge" not in size:
            raise ValueError(f"preprocessor_config.json: size={size!r}; only a shortest_edge resize is implemented")
        size = size["shortest_edge"]
    crop = _edge(raw, "crop_size", 224)
    if isinstance(crop, dict):
        if "height" not in crop or "width" not in crop:
            raise ValueError(f"preprocessor_config.json: crop_size={crop!r} needs height and width")
        crop_h, crop_w = crop["height"], crop["width"]
    else:
        crop_h = crop_w = crop
    if crop_h > size or crop_w > size:
        raise ValueError(f"preprocessor_config.json: crop_size {crop_h}x{crop_w} is larger than size {size}")
    mean = tuple(float(v) for v in raw.get("image_mean", OPENAI_CLIP_MEAN))
    std = tuple(float(v) for v in raw.get("image_std", OPENAI_CLIP_STD))
    for key, v in (("image_mean", mean), ("image_std", std)):
        if len(v) != 3:
            raise ValueError(f"preprocessor_config.json: {key} has {len(v)} entries, expected 3")
    return dict(size=int(size), crop_h=int(crop_h), crop_w=int(crop_w), mean=mean, std=std)


def load_safety_checker(model_dir: str):
    """``<model_dir>/safety_checker/`` and ``<model_dir>/feature_extractor/`` -> (config, state dict, preprocessing
    config).  A checker without a feature extractor raises."""
    fe = os.path.join(model_dir, "feature_extractor", "preprocessor_config.json")
    if not os.path.exists(fe):
        raise FileNotFoundError(f"{model_dir} has a safety_checker/ but no feature_extractor/preprocessor_config.json")
    with open(os.path.join(model_dir, "safety_checker", "config.json")) as f:
        cfg = C.safety_checker_config(json.load(f))
    with open(fe) as f:
        pre = preprocessor_config(json.load(f))
    return cfg, load_component(model_dir, "safety_checker", cfg), pre
