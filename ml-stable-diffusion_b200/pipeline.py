"""Text-to-image pipeline with the reference's call surface, running on the sm_90a kernels.

Mirrors ``CoreMLStableDiffusionPipeline.__call__`` (``python_coreml_stable_diffusion/pipeline.py:403-589``):
same keyword arguments, same order of operations (encode -> latents -> [CFG-duplicated UNet ->
guidance -> scheduler.step] x N -> VAE decode -> clip -> NHWC -> PIL), same
``StableDiffusionPipelineOutput(images, nsfw_content_detected)`` result.  Differences, all by design:

* the loop body stays on the GPU: UNet (CUDA graph), then ONE fused kernel for guidance + scheduler
  step; there is no per-step host round trip (the reference crosses numpy<->Core ML twice per step);
* batches of prompts are accepted (the reference raises ``NotImplementedError``, pipeline.py:434-438;
  BASELINE config 3 needs 8 prompts per GPU);
* the CLIP text encoder / tokenizer are not part of this round's hot path (SURVEY 8f N2): prompts
  are turned into *synthetic* 77-token embeddings by ``SyntheticTextEncoder`` unless the caller
  passes ``prompt_embeds`` or installs a real ``text_encoder`` callable with the reference contract
  (``input_ids`` float32 (1, 77) -> ``last_hidden_state`` (1, 77, D), pipeline.py:151-175).
"""
from __future__ import annotations

import dataclasses
import hashlib
from typing import List, Optional, Tuple, Union

import numpy as np
import torch

from . import config as C
from . import lib as L
from . import scheduler as S
from .model import UNetModel
from .unet import ControlResiduals
from .vae import VAEDecoderModel


def vae_dtype(unet_cfg: dict, vae_cfg: dict):
    """The VAE's activation type for a checkpoint: bf16 iff the UNet is SDXL's (``addition_embed_type ==
    "text_time"``) and the VAE's config sets ``"force_upcast": true`` -- the stock SDXL VAE, whose decoder activations
    exceed fp16's range (diffusers upcasts exactly these VAEs in its SDXL pipeline; the reference converts the XL VAE
    in FLOAT32 unless a custom VAE is given).  A missing key counts as false, so the fp16-fix VAE and every SD 1.x /
    2.x directory keep fp16.  The checkpoint decides; there is no switch."""
    xl = unet_cfg.get("addition_embed_type") == "text_time"
    return torch.bfloat16 if xl and vae_cfg.get("force_upcast") is True else torch.float16


#: the schedulers whose truncated schedule (inpainting at strength < 1) diffusers 0.30.2 runs as ``plan(start)``
INPAINT_STRENGTH_SCHEDULERS = ("DDIM", "DPMSolverMultistep")


def _per_net(value, n_nets, name):
    """A float, or one per ControlNet -> list of n_nets floats (ValueError naming ``name`` on a wrong length)."""
    vals = list(value) if isinstance(value, (list, tuple, np.ndarray)) else [value] * n_nets
    if len(vals) != n_nets:
        raise ValueError(f"{name} has {len(vals)} values for {n_nets} ControlNet(s)")
    return [float(v) for v in vals]


def controlnet_arguments(n_nets, controlnet_conditioning_scale=1.0, control_guidance_start=0.0,
                         control_guidance_end=1.0, guess_mode=False):
    """Checks the ControlNet arguments of ``__call__`` as diffusers' check_inputs does -> (scales, starts, ends), one
    float per net.  Scales must be finite; every window must satisfy 0 <= start < end <= 1.  guess_mode is not
    implemented."""
    if guess_mode:
        raise ValueError("guess_mode=True is not implemented")
    scales = _per_net(controlnet_conditioning_scale, n_nets, "controlnet_conditioning_scale")
    if not all(np.isfinite(scales)):
        raise ValueError(f"controlnet_conditioning_scale must be finite, got {scales}")
    starts = _per_net(control_guidance_start, n_nets, "control_guidance_start")
    ends = _per_net(control_guidance_end, n_nets, "control_guidance_end")
    for s, e in zip(starts, ends):
        if not (0.0 <= s < e <= 1.0):
            raise ValueError(f"control_guidance_start / control_guidance_end: need 0 <= start < end <= 1, got start={s} "
                             f"end={e}")
    return scales, starts, ends


def controlnet_keep(n_steps, starts, ends):
    """diffusers' controlnet_keep over the ``n_steps`` executed steps (after an image-to-image start): net k runs at
    step i unless i / n_steps < start_k or (i + 1) / n_steps > end_k.  -> per step, the tuple of the nets that run."""
    return [tuple(k for k, (s, e) in enumerate(zip(starts, ends)) if not (i / n_steps < s or (i + 1) / n_steps > e))
            for i in range(n_steps)]


def prepare_mask_and_masked_image(image, mask):
    """diffusers 0.30.2 ``StableDiffusionInpaintPipeline``'s mask processing (``VaeImageProcessor(do_binarize=True,
    do_convert_grayscale=True)``): ``image`` (B, 3, H, W) in [-1, 1]; ``mask`` (B | 1, 1, H, W) or (H, W) in [0, 1],
    1 = repaint.  The mask is binarised at 0.5 (0.5 repaints) and broadcast to B; the masked image is
    ``image * (mask < 0.5)``.  -> (mask (B, 1, H, W) float32 in {0, 1}, masked image (B, 3, H, W) float32)."""
    image = np.asarray(image, dtype=np.float32)
    if image.ndim != 4 or image.shape[1] != 3:
        raise ValueError(f"starting_image must be (B, 3, H, W), got shape {image.shape}")
    m = np.asarray(mask, dtype=np.float32)
    if m.ndim == 2:
        m = m[None, None]
    if m.ndim != 4 or m.shape[1] != 1:
        raise ValueError(f"mask_image must be (B, 1, H, W), (1, 1, H, W) or (H, W), got shape {np.shape(mask)}")
    if m.shape[2:] != image.shape[2:]:
        raise ValueError(f"mask_image is {m.shape[2]}x{m.shape[3]}, the starting image {image.shape[2]}x{image.shape[3]}")
    if m.shape[0] not in (1, image.shape[0]):
        raise ValueError(f"mask_image has batch {m.shape[0]}, the starting image {image.shape[0]}")
    if not (np.isfinite(m).all() and m.min() >= 0.0 and m.max() <= 1.0):
        raise ValueError("mask_image values must lie in [0, 1]")
    m = np.broadcast_to((m >= 0.5).astype(np.float32), (image.shape[0], 1) + image.shape[2:])
    return np.ascontiguousarray(m), image * (m < 0.5)


def latent_mask(mask, factor=8):
    """``F.interpolate(mask, size=(H // factor, W // factor))`` (nearest, the inpaint pipeline's default): latent
    pixel (i, j) takes image pixel (factor i, factor j)."""
    return np.ascontiguousarray(np.asarray(mask, dtype=np.float32)[:, :, ::factor, ::factor])


@dataclasses.dataclass
class InpaintInputs:
    """One inpainting call's inputs to ``denoise`` (numpy or torch, float32): ``mask`` the latent mask (n, 1, h, w) in
    {0, 1}, 1 = repaint; for a 4-channel UNet ``image_latents`` (the encoded image x0_img, x-space) and ``noise`` (the
    initial noise z, unscaled), which the blend reads; for a 9-channel UNet ``masked_image_latents``."""
    mask: object
    image_latents: object = None
    noise: object = None
    masked_image_latents: object = None


@dataclasses.dataclass
class StableDiffusionPipelineOutput:
    images: Union[List, np.ndarray]
    nsfw_content_detected: Optional[List[bool]]


class SyntheticTokenizer:
    """Deterministic stand-in for the CLIP BPE tokenizer: whitespace words -> ids by hash, padded to
    ``model_max_length`` with the end-of-text id (same padding convention as pipeline.py:151-158)."""
    model_max_length = 77
    bos, eos, vocab = 49406, 49407, 49408

    def __call__(self, text: str):
        ids = [self.bos]
        for wd in text.lower().split()[: self.model_max_length - 2]:
            ids.append(int.from_bytes(hashlib.sha256(wd.encode()).digest()[:4], "little") % (self.bos - 1) + 1)
        ids.append(self.eos)
        ids += [self.eos] * (self.model_max_length - len(ids))
        return np.array([ids], dtype=np.float32)  # the reference feeds input_ids as float32 (pipeline.py:173)


class SyntheticTextEncoder:
    """Maps token ids to fixed pseudo-random unit-variance embeddings (no weights exist offline)."""

    def __init__(self, hidden=1024, seq=77):
        self.hidden, self.seq = hidden, seq
        self.expected_inputs = {"input_ids": {"shape": (1, seq), "dtype": np.dtype(np.float32)}}

    def __call__(self, input_ids):
        out = np.empty((1, self.seq, self.hidden), dtype=np.float32)
        for i, tok in enumerate(np.asarray(input_ids).reshape(-1).astype(np.int64)):
            out[0, i] = np.random.RandomState(int(tok) * 131 + i).standard_normal(self.hidden)
        return {"last_hidden_state": out}


class B200StableDiffusionPipeline:
    """Drop-in for ``CoreMLStableDiffusionPipeline`` on one H100."""

    def __init__(self, unet: UNetModel, vae_decoder: VAEDecoderModel, scheduler="DDIM", text_encoder=None,
                 tokenizer=None, force_zeros_for_empty_prompt=True, xl=False, controlnet=None, loop_graph=True,
                 vae_encoder=None, text_encoder_2=None, tokenizer_2=None, scheduler_kwargs=None, unet_refiner=None,
                 safety_checker=None):
        self.unet = unet
        # safety_checker.SafetyCheckerEngine or None: runs after the VAE decode, on the device (pipeline.py:286-311)
        self.safety_checker = safety_checker
        # SDXL refiner UNet (StableDiffusionXLPipeline.swift:205-225): takes over the loop at step
        # int(len(timesteps) * refiner_start) with its own conditioning (set_refiner_inputs)
        self.unet_refiner = unet_refiner
        self.text_encoder_2 = text_encoder_2  # SDXL: CLIPTextModelWithProjection slot (pipeline.py:64-65, 136-141)
        self.tokenizer_2 = tokenizer_2
        self.vae_encoder = vae_encoder  # VAEEncoderModel or None (image-to-image, StableDiffusionPipeline.swift:371-376)
        self.loop_graph = bool(loop_graph) and unet.use_cuda_graph  # whole-loop CUDA graph (denoise())
        self._loop_graphs = {}
        self.controlnet = list(controlnet) if controlnet else None  # pipeline.py:66,106: Optional[List[model]]
        if self.controlnet and not unet.engine.support_controlnet:
            raise ValueError("the UNet was not built with support_controlnet=True (no additional_residual inputs)")
        if self.controlnet:
            if unet_refiner is not None:
                raise ValueError("ControlNet cannot be combined with the SDXL refiner")
            if len(self.controlnet) > L.MAX_CONTROLNETS:
                raise ValueError(f"at most {L.MAX_CONTROLNETS} ControlNets, got {len(self.controlnet)}")
            for k, net in enumerate(self.controlnet):
                C.check_controlnet_matches_unet(unet.engine.cfg, net.engine.cfg, f"ControlNet {k}")
            # conditioning scales on the device, one fp32 array per set of nets that runs at some step (the loop graph
            # reads them, so a new scale replays the same graph); the set of all nets exists from the start
            self._all_nets = tuple(range(len(self.controlnet)))
            self._control_scale_bufs = {self._all_nets: torch.ones(len(self.controlnet), dtype=torch.float32,
                                                                   device=unet.device)}
        self.vae_decoder = vae_decoder
        self.scheduler_name = scheduler
        # this class mirrors the reference's PYTHON pipeline, whose DPM-Solver++ is diffusers 0.30.2
        # (final_sigmas_type="zero"); pass scheduler_kwargs={"final_sigmas_type": "sigma_min"} for the Swift CLI's ending
        self.scheduler_kwargs = dict(scheduler_kwargs or {})
        if scheduler == "DPMSolverMultistep":
            self.scheduler_kwargs.setdefault("final_sigmas_type", "zero")
        self.device = unet.device
        self.xl = xl
        d_ctx = unet.engine.cfg["cross_attention_dim"]
        self.text_encoder = text_encoder or SyntheticTextEncoder(d_ctx, unet.seq)
        self.tokenizer = tokenizer or SyntheticTokenizer()
        self.force_zeros_for_empty_prompt = force_zeros_for_empty_prompt
        self.vae_scale_factor = vae_decoder.scale
        self.height = unet.h * self.vae_scale_factor
        self.width = unet.w * self.vae_scale_factor
        self.images_per_call = unet.batch // 2
        # the latents have the UNet's OUTPUT channels: an inpainting UNet reads 9 (latents, mask, masked image latents)
        self.latent_channels = unet.engine.out_ch
        n, c, h, w = self.images_per_call, self.latent_channels, unet.h, unet.w
        dev = self.device
        self._latents = torch.zeros(n, c, h, w, dtype=torch.float32, device=dev)
        self._hist = torch.zeros(4, n, c, h, w, dtype=torch.float32, device=dev)
        self._denoised = torch.zeros(n, c, h, w, dtype=torch.float32, device=dev)
        self._ctx = torch.zeros(2 * n, d_ctx, 1, unet.seq, dtype=torch.float16, device=dev)
        self._t = torch.zeros(2 * n, dtype=torch.float32, device=dev)
        # ancestral samplers: Philox key of the step noise (filled before each loop, so one loop graph serves every
        # seed) and the draw number of step 0 (part of the graph key: offsets are baked into the graph)
        self._noise_key = torch.zeros(1, dtype=torch.int32, device=dev)
        self._noise_base = 0
        # inpainting: static device buffers (allocated on first use), filled before each loop so that one loop graph
        # serves every mask, image and seed
        self._inpaint_bufs = None

    # ---------------------------------------------------------------- factory
    @classmethod
    def from_random_init(cls, model_version="sd21-base", images_per_call=1, device="cuda", seed=0,
                         scheduler="DDIM", height=None, width=None, unet_cfg=None, vae_cfg=None, controlnet_cfgs=None,
                         text_encoder_cfg=None, tokenizer=None, with_vae_encoder=False, scheduler_kwargs=None,
                         safety_checker_cfg=None):
        """Random-init weights of the named architecture (no checkpoints exist offline).  ``controlnet_cfgs``:
        list of ControlNet configs (seeded seed+2, seed+3, ...); switches the UNet to its control variant.
        ``model_version``: "sd21-base", "sd21" (SD 2.0 / 2.1 768-v: 768x768 by default, v-prediction), "sd15"
        (SD 1.4 / 1.5), "sdxl-base" or "tiny"; ``height`` / ``width`` default to 768 for "sd21" and 512 otherwise.
        ``text_encoder_cfg``: a CLIP text config (config.OPENCLIP_H_TEXT for SD-2.x, config.CLIP_L_TEXT for SD-1.x) -> the
        text encoder runs on the
        device (random-init, seed+100) instead of the synthetic embedding table; ``tokenizer``: e.g. a
        ``tokenizer.BPETokenizer`` built from the checkpoint's vocab.json / merges.txt.  ``scheduler_kwargs``: extra
        scheduler arguments (e.g. ``{"prediction_type": "v_prediction"}``, the default for "sd21").
        ``safety_checker_cfg``: e.g. config.SD_SAFETY_CHECKER -> a random-init safety checker (seed+200) with
        CLIPImageProcessor's default preprocessing."""
        native = 768 if model_version == "sd21" else 512
        height, width = height or native, width or native
        scheduler_kwargs = dict(scheduler_kwargs or {})
        if model_version == "sd21":
            if scheduler not in S.PREDICTION_TYPE_SCHEDULERS:
                raise ValueError(f"the sd21 (768-v) model is a v-prediction model; the {scheduler} scheduler runs "
                                 f"epsilon prediction only (use one of {S.PREDICTION_TYPE_SCHEDULERS})")
            scheduler_kwargs.setdefault("prediction_type", "v_prediction")
        unet_cfg = unet_cfg or {"sd21-base": C.SD21_BASE_UNET, "sd21": C.SD21_UNET, "sd15": C.SD15_UNET,
                                "sdxl-base": C.SDXL_BASE_UNET, "tiny": C.TINY_UNET}[model_version]
        vae_cfg = vae_cfg or (C.TINY_VAE if model_version == "tiny" else C.SD_VAE)
        if controlnet_cfgs:
            unet_cfg = dict(unet_cfg, support_controlnet=True)
        f = 2 ** (len(vae_cfg["block_out_channels"]) - 1)
        usd = C.random_state_dict(C.unet_param_shapes(unet_cfg), seed=seed, dtype=torch.float16)
        vsd = C.random_state_dict(C.vae_decoder_param_shapes(vae_cfg), seed=seed + 1, dtype=torch.float16)
        unet = UNetModel(unet_cfg, usd, batch=2 * images_per_call, height=height // f, width=width // f,
                         device=device)
        vae = VAEDecoderModel(vae_cfg, vsd, batch=images_per_call, height=height // f, width=width // f,
                              device=device)
        nets = None
        if controlnet_cfgs:
            from .controlnet import ControlNetModel
            nets = [ControlNetModel(c, C.random_state_dict(C.controlnet_param_shapes(c), seed=seed + 2 + i,
                                                           dtype=torch.float16),
                                    batch=2 * images_per_call, height=height // f, width=width // f, device=device)
                    for i, c in enumerate(controlnet_cfgs)]
        enc = None
        if text_encoder_cfg is not None:
            from .text_encoder import TextEncoderModel
            if text_encoder_cfg["hidden_size"] != unet_cfg["cross_attention_dim"]:
                raise ValueError("text encoder width does not match the UNet's cross_attention_dim")
            enc = TextEncoderModel(text_encoder_cfg, C.random_clip_text_state_dict(text_encoder_cfg, seed=seed + 100,
                                                                                   dtype=torch.float16),
                                   batch=1, device=device)
        venc = None
        if with_vae_encoder:
            from .vae import VAEEncoderModel
            esd = C.random_state_dict(C.vae_encoder_param_shapes(vae_cfg), seed=seed + 50, dtype=torch.float16)
            venc = VAEEncoderModel(vae_cfg, esd, batch=images_per_call, height=height, width=width, device=device)
        checker = None
        if safety_checker_cfg is not None:
            from .safety_checker import SafetyCheckerEngine
            checker = SafetyCheckerEngine(safety_checker_cfg, C.random_safety_checker_state_dict(
                safety_checker_cfg, seed=seed + 200, dtype=torch.float16), device=device)
        return cls(unet, vae, scheduler=scheduler, xl=unet.engine.xl, controlnet=nets, text_encoder=enc,
                   tokenizer=tokenizer, vae_encoder=venc, force_zeros_for_empty_prompt=unet.engine.xl,
                   scheduler_kwargs=scheduler_kwargs, safety_checker=checker)

    _SCHEDULER_CLASS = {"PNDMScheduler": "PNDM", "DDIMScheduler": "DDIM", "DPMSolverMultistepScheduler": "DPMSolverMultistep",
                        "LCMScheduler": "LCM", "EulerDiscreteScheduler": "EulerDiscrete",
                        "EulerAncestralDiscreteScheduler": "EulerAncestralDiscrete",
                        "LMSDiscreteScheduler": "LMSDiscrete"}

    @classmethod
    def scheduler_from_config(cls, sched_cfg: dict) -> str:
        """The scheduler a checkpoint's ``scheduler_config.json`` names (``_class_name``, PNDM when absent).  The Euler /
        Euler-ancestral / LMS classes are taken from the checkpoint only with the ``"trailing"`` spacing the few-step
        checkpoints ship (SD-Turbo, SDXL-Turbo, SDXL-Lightning); with any other spacing (SDXL-base's ``"leading"``
        Euler) the caller chooses the sampler through ``scheduler_override``, as before."""
        name = sched_cfg.get("_class_name", "PNDMScheduler")
        sched = cls._SCHEDULER_CLASS.get(name)
        if sched is None or (sched in S.SIGMA_SCHEDULERS and sched_cfg.get("timestep_spacing") != "trailing"):
            why = "" if sched is None else f" with timestep_spacing={sched_cfg.get('timestep_spacing')!r}"
            raise ValueError(f"scheduler {name} of the checkpoint{why} is not implemented as its default; pass "
                             f"scheduler_override (one of {sorted(S.SCHEDULER_MAP)})")
        return sched

    def do_classifier_free_guidance(self, guidance_scale):
        """diffusers' rule: classifier-free guidance runs iff guidance_scale > 1 and the UNet has no guidance
        embedding (time_cond_proj_dim).  Otherwise the loop runs guidance-free, the UNet on the N prompt rows only."""
        return guidance_scale > 1.0 and not self.unet.engine.time_cond_dim

    @classmethod
    def from_pretrained(cls, model_dir, images_per_call=1, device="cuda", height=None, width=None,
                        scheduler_override=None, controlnet_dirs=None, force_zeros_for_empty_prompt=None,
                        with_vae_encoder=False, refiner_dir=None, load_safety_checker=True, unet_quantization=None,
                        unet_palettization=None):
        """Build the pipeline from a diffusers-layout model directory (``unet/``, ``vae/``, ``text_encoder[_2]/``,
        ``tokenizer[_2]/``, ``scheduler/``): the counterpart of ``get_coreml_pipe(pytorch_pipe, mlpackages_dir,
        model_version, compute_unit, scheduler_override, controlnet_models, force_zeros_for_empty_prompt)``
        (pipeline.py:607-697), which wires converted .mlpackage files to the same slots.  Weights are read with
        ``checkpoint.load_component`` (schema-checked), configs with ``checkpoint.read_config``.
        ``refiner_dir``: an SDXL refiner directory whose UNet takes over at ``refiner_start`` (``__call__``).
        ``load_safety_checker``: load ``safety_checker/`` with ``feature_extractor/`` when the directory has them (SD 1.4
        / 1.5; get_coreml_pipe loads it whenever the diffusers pipeline has one, pipeline.py:650-656); False skips it.
        ``unet_quantization``: a ``quantization.W8A8Recipe`` or the path of a saved one (``calibrate_unet``); the base
        UNet runs the convolutions it names in W8A8.  The refiner, ControlNets, VAE and text encoders stay fp16.
        ``unet_palettization``: n-bit palettized base-UNet weights -- an nbits int, a {layer: nbits} dict or
        (pre-analysis json path, recipe key) (``palettization.as_recipe``); the same components stay fp16."""
        import json
        import os
        from . import checkpoint as K
        from .text_encoder import TextEncoderModel
        from .tokenizer import BPETokenizer

        ucfg = K.read_config(model_dir, "unet")
        vcfg = K.read_config(model_dir, "vae")
        ccfgs = []
        if controlnet_dirs:
            if refiner_dir:
                raise ValueError("ControlNet cannot be combined with the SDXL refiner")
            for k, d in enumerate(controlnet_dirs):  # checked before any weights are read
                with open(os.path.join(d, "config.json")) as fh:
                    ccfg = {k2: (tuple(v) if isinstance(v, list) else v) for k2, v in json.load(fh).items()
                            if not k2.startswith("_")}
                C.check_controlnet_matches_unet(ucfg, ccfg, f"ControlNet {k} ({d})")
                ccfgs.append(ccfg)
            ucfg = dict(ucfg, support_controlnet=True)
        f = 2 ** (len(vcfg["block_out_channels"]) - 1)
        size = ucfg.get("sample_size", 64)
        h = (height // f) if height else size
        w = (width // f) if width else size
        xl = ucfg.get("addition_embed_type") == "text_time"
        unet = UNetModel(ucfg, K.load_component(model_dir, "unet", ucfg), batch=2 * images_per_call, height=h, width=w,
                         device=device, quantization=unet_quantization, palettization=unet_palettization)
        vsd = K.read_state_dict(os.path.join(model_dir, "vae"))
        vdtype = vae_dtype(ucfg, vcfg)
        vae = VAEDecoderModel(vcfg, K.check_state_dict("vae_decoder", vcfg, vsd), batch=images_per_call, height=h,
                              width=w, device=device, dtype=vdtype)
        venc = None
        if with_vae_encoder:
            from .vae import VAEEncoderModel
            venc = VAEEncoderModel(vcfg, K.check_state_dict("vae_encoder", vcfg, vsd), batch=images_per_call,
                                   height=h * f, width=w * f, device=device, dtype=vdtype)

        def text_pair(enc_dir, tok_dir):
            if not os.path.isdir(os.path.join(model_dir, enc_dir)):
                return None, None
            tcfg = K.read_config(model_dir, enc_dir)
            # SDXL conditions on hidden_states[-2] of both encoders (torch2coreml.py:416-446: ``hidden_embeds``)
            enc = TextEncoderModel(tcfg, K.load_component(model_dir, enc_dir, tcfg), batch=1, device=device,
                                   hidden_layer=-2 if xl else None)
            tok = None
            tdir = os.path.join(model_dir, tok_dir)
            if os.path.exists(os.path.join(tdir, "merges.txt")):
                pad = "<|endoftext|>"
                stm = os.path.join(tdir, "special_tokens_map.json")  # SDXL's second tokenizer pads with "!"
                if os.path.exists(stm):
                    with open(stm) as fh:
                        pt = json.load(fh).get("pad_token", pad)
                    pad = pt.get("content", pad) if isinstance(pt, dict) else pt
                tok = BPETokenizer.from_files(os.path.join(tdir, "merges.txt"), os.path.join(tdir, "vocab.json"), pad_token=pad)
            return enc, tok

        enc1, tok1 = text_pair("text_encoder", "tokenizer")
        enc2, tok2 = text_pair("text_encoder_2", "tokenizer_2")
        sched = scheduler_override
        sched_kw = None
        sched_cfg = os.path.join(model_dir, "scheduler", "scheduler_config.json")
        if sched is None:
            with open(sched_cfg) as fh:
                sched = cls.scheduler_from_config(json.load(fh))
        if sched in S.SIGMA_SCHEDULERS + ("LCM",) and os.path.exists(sched_cfg):
            # SCHEDULER_MAP[name].from_config(pytorch_pipe.scheduler.config) (pipeline.py:672-676): spacing, offset
            # and betas come from the checkpoint (SDXL: "leading", offset 1; Turbo / Lightning: "trailing")
            with open(sched_cfg) as fh:
                sc = json.load(fh)
            sched_kw = S.lcm_scheduler_kwargs(sc) if sched == "LCM" else S.sigma_scheduler_kwargs(sc)
        if sched in S.PREDICTION_TYPE_SCHEDULERS and os.path.exists(sched_cfg):
            # SD 2.0 / 2.1 768-v checkpoints are v-prediction models ("prediction_type": "v_prediction"); diffusers
            # applies the key inside scheduler.step (pipeline.py:565-569), these schedulers take it in their plan
            with open(sched_cfg) as fh:
                pred = json.load(fh).get("prediction_type")
            if pred is not None:
                sched_kw = {"prediction_type": S.check_prediction_type(pred)}
        nets = None
        if controlnet_dirs:
            from .controlnet import ControlNetModel
            nets = []
            for d, ccfg in zip(controlnet_dirs, ccfgs):
                nets.append(ControlNetModel(ccfg, K.load_component(d, "controlnet", ccfg), batch=2 * images_per_call,
                                            height=h, width=w, device=device))
        refiner = None
        if refiner_dir:
            rcfg = K.read_config(refiner_dir, "unet")
            # the refiner's config.json names add_embedding's input width (2560) but not its five time ids; the rows
            # __call__ builds for it are five wide, so the count comes from the width its pooled embedding leaves
            pooled = C.SDXL_POOLED_DIM
            enc2 = os.path.join(refiner_dir, "text_encoder_2", "config.json")
            if os.path.exists(enc2):
                with open(enc2) as fh:
                    pooled = json.load(fh).get("projection_dim", pooled)
            rcfg = dict(rcfg, num_time_ids=C.num_time_ids(rcfg, pooled))
            refiner = UNetModel(rcfg, K.load_component(refiner_dir, "unet", rcfg), batch=2 * images_per_call, height=h,
                                width=w, device=device)
        if force_zeros_for_empty_prompt is None:
            force_zeros_for_empty_prompt = xl   # the reference's CLI sets it for SDXL only (pipeline.py:744-755)
        checker = None
        if load_safety_checker and os.path.isdir(os.path.join(model_dir, "safety_checker")):
            from .safety_checker import SafetyCheckerEngine
            checker = SafetyCheckerEngine(*K.load_safety_checker(model_dir), device=device)
        return cls(unet, vae, scheduler=sched, text_encoder=enc1, tokenizer=tok1, text_encoder_2=enc2, tokenizer_2=tok2,
                   xl=xl, controlnet=nets, vae_encoder=venc, force_zeros_for_empty_prompt=force_zeros_for_empty_prompt,
                   unet_refiner=refiner, scheduler_kwargs=sched_kw, safety_checker=checker)

    # ---------------------------------------------------------------- reference-named helpers
    def check_inputs(self, prompt, height, width, callback_steps):
        """pipeline.py:359-382."""
        if not isinstance(prompt, (str, list)):
            raise ValueError(f"`prompt` has to be of type `str` or `list` but is {type(prompt)}")
        if height % 8 != 0 or width % 8 != 0:
            raise ValueError(f"`height` and `width` have to be divisible by 8 but are {height} and {width}.")
        if callback_steps is None or not isinstance(callback_steps, int) or callback_steps <= 0:
            raise ValueError(f"`callback_steps` has to be a positive integer but is {callback_steps} of type "
                             f"{type(callback_steps)}.")

    def _encode_one(self, text):
        ids = self.tokenizer(text)
        return np.asarray(self.text_encoder(input_ids=ids)["last_hidden_state"], dtype=np.float32)[0]  # (S, D)

    def _encode_prompt(self, prompts, do_cfg, negative_prompt):
        """-> (2B, D, 1, S) fp16 array, uncond half first (pipeline.py:123-257: concat [neg, pos], :252 transpose)."""
        conds = [self._encode_one(p) for p in prompts]
        if isinstance(negative_prompt, list):
            if len(negative_prompt) != len(prompts):
                raise ValueError(f"`negative_prompt` has batch size {len(negative_prompt)}, but `prompt` has batch size "
                                 f"{len(prompts)}")
            negs = list(negative_prompt)
        else:
            negs = [negative_prompt] * len(prompts)
        unconds = []
        for ng, cnd in zip(negs, conds):
            if not do_cfg:
                unconds.append(cnd)
            elif ng is None and self.force_zeros_for_empty_prompt:
                # pipeline.py:183-184: zeros only when NO negative prompt was given and the flag is set (the
                # reference's CLI sets it for SDXL only, pipeline.py:744-755); an explicit "" is encoded
                unconds.append(np.zeros_like(cnd))
            else:
                unconds.append(self._encode_one(ng or ""))
        emb = np.stack(unconds + conds, 0)  # (2B, S, D)
        return np.ascontiguousarray(emb.transpose(0, 2, 1)[:, :, None, :]).astype(np.float16)

    def _encode_prompt_xl(self, prompts, do_cfg, negative_prompt=None, prompts_2=None, negative_prompt_2=None,
                          only_second=False):
        """SDXL branch of pipeline.py:123-257: both encoders' ``hidden_embeds`` concatenated along the feature axis
        (encoder 1 first), the pooled output of the LAST encoder, zeros for the negative branch when no negative
        prompt is given and force_zeros_for_empty_prompt.  The refiner has only encoder 2 (text_encoder is None).
        -> ((2B, D1 + D2, 1, S) fp16, (2B, P) fp32), uncond half first."""
        pairs = [(self.tokenizer, self.text_encoder), (self.tokenizer_2, self.text_encoder_2)]
        if self.text_encoder is None or only_second:  # the refiner is conditioned on the second encoder only
            pairs = pairs[1:]
        texts = [prompts, prompts_2 if prompts_2 is not None else prompts][-len(pairs):]

        def run(text_lists):
            per_prompt, pooled = [], []
            for i in range(len(text_lists[0])):
                feats = []
                for (tok, enc), tl in zip(pairs, text_lists):
                    o = enc(input_ids=np.asarray(tok(tl[i]), dtype=np.float32))
                    feats.append(np.asarray(o["hidden_embeds"], dtype=np.float32)[0])
                    last_pooled = np.asarray(o["pooled_outputs"], dtype=np.float32)[0]
                per_prompt.append(np.concatenate(feats, axis=-1))  # (S, D1 + D2)
                pooled.append(last_pooled)
            return np.stack(per_prompt, 0), np.stack(pooled, 0)

        emb, pooled = run(texts)
        if do_cfg:
            if negative_prompt is None and self.force_zeros_for_empty_prompt:
                neg, neg_pooled = np.zeros_like(emb), np.zeros_like(pooled)
            else:
                neg_1 = negative_prompt or ""
                neg_2 = negative_prompt_2 or neg_1
                as_list = lambda v: [v] * len(prompts) if isinstance(v, str) else list(v)  # noqa: E731
                neg_1, neg_2 = as_list(neg_1), as_list(neg_2)
                if len(neg_1) != len(prompts):
                    raise ValueError(f"`negative_prompt` has batch size {len(neg_1)}, but `prompt` has batch size "
                                     f"{len(prompts)}")
                neg, neg_pooled = run([neg_1, neg_2][-len(pairs):])
            emb, pooled = np.concatenate([neg, emb], 0), np.concatenate([neg_pooled, pooled], 0)
        else:
            # the UNet always runs both batch halves: without guidance both carry the prompt (like _encode_prompt)
            emb, pooled = np.concatenate([emb, emb], 0), np.concatenate([pooled, pooled], 0)
        return np.ascontiguousarray(emb.transpose(0, 2, 1)[:, :, None, :]).astype(np.float16), pooled

    def prepare_latents(self, batch, channels, height, width, latents=None, seed=None, rng="numpy",
                        init_noise_sigma=1.0):
        """pipeline.py:322-344: np.random.randn(...).astype(fp16) * init_noise_sigma (the global numpy stream, seeded by
        the caller like pipeline.py:725-726).  With ``seed``: the Swift pipeline's ``generateLatentSamples``
        (StableDiffusionPipeline.swift:361-379): one draw of C*h*w normals per image from the chosen
        ``StableDiffusionRNG`` source (numpy / torch / nvidia, rng.py), so a seed reproduces the reference CLIs' latents.
        ``init_noise_sigma``: the scheduler's (1 for DDIM / DPM-Solver++ / PNDM, sigma_max or sqrt(sigma_max^2 + 1) for
        the Euler / LMS samplers)."""
        shape = (batch, channels, height // self.vae_scale_factor, width // self.vae_scale_factor)
        if latents is None and seed is not None:
            from .rng import random_source
            src = random_source(rng, seed)
            per = int(np.prod(shape[1:]))
            latents = np.stack([src.normal_array(per).reshape(shape[1:]) for _ in range(batch)]).astype(np.float32)
        elif latents is None:
            latents = np.random.randn(*shape).astype(np.float16)
        elif tuple(latents.shape) != shape:
            raise ValueError(f"Unexpected latents shape, got {latents.shape}, expected {shape}")
        return latents.astype(np.float32) * init_noise_sigma

    def prepare_control_cond(self, controlnet_cond, do_classifier_free_guidance, batch_size, num_images_per_prompt):
        """pipeline.py:345-356: each (3, H, W) condition image is repeated per image and doubled for CFG."""
        out = []
        for cond in controlnet_cond:
            cond = np.stack([np.asarray(cond)] * batch_size * num_images_per_prompt)
            # doubled like the latents: this engine always runs both batch halves (with guidance <= 1 both carry the
            # prompt), where the reference doubles only under guidance (pipeline.py:345-356)
            cond = np.concatenate([cond] * 2)
            out.append(cond)
        return out

    def run_controlnet(self, sample, timestep, encoder_hidden_states, controlnet_cond, nets=None, time_ids=None,
                       text_embeds=None):
        """pipeline.py:259-284 on the device: every ControlNet in ``nets`` (indices; default all) sees the same UNet
        inputs (``time_ids`` / ``text_embeds``: those of an SDXL UNet); their residuals are scaled and summed in
        diffusers' fp16 order (one launch per residual, the scales of ``_control_scale_bufs[nets]``).  Returns NCHW
        views of NHWC fp16 tensors, or None when ``nets`` is empty."""
        if not self.controlnet:
            raise ValueError("Conditions for controlnet are given but the pipeline has no controlnet modules")
        nets = self._all_nets if nets is None else tuple(nets)
        if not nets:
            return None
        r = sample.shape[0]  # the batch, or its first half in the guidance-free loop
        outs = []
        for k in nets:
            module, cond = self.controlnet[k], controlnet_cond[k]
            module._sample[:r].copy_(sample)
            module._t[:r].copy_(timestep)
            module._ctx[:r].copy_(encoder_hidden_states)
            module._cond[:r].copy_(cond)
            if module.engine.xl:
                module._time_ids[:r].copy_(torch.as_tensor(time_ids).reshape(r, -1))
                module._text_embeds[:r].copy_(torch.as_tensor(text_embeds))
            outs.append(module.forward_device(r))
        scales = self._control_scale_bufs[nets]
        total = [L.control_inject(None, [o[i] for o in outs], scales) for i in range(len(outs[0]))]
        return [t.permute(0, 3, 1, 2) for t in total]

    @staticmethod
    def numpy_to_pil(images):
        from PIL import Image
        images = (images * 255).round().astype("uint8")
        return [Image.fromarray(im) for im in images]

    # ---------------------------------------------------------------- device loop
    @staticmethod
    def _coeffs(st, guidance_scale, k=None):
        k = k or L.StepCoeffs()
        k.guidance = float(guidance_scale)
        k.cx, k.ce, k.x0_cx, k.x0_ce = st.cx, st.ce, st.x0_cx, st.x0_ce
        for j in range(4):
            k.ch[j] = st.ch[j]
            k.x0_ch[j] = st.x0_ch[j]
        k.n_hist, k.push_eps_slot, k.push_x0_slot, k.push_x_slot = (st.n_hist, st.push_eps_slot,
                                                                    st.push_x0_slot, st.push_x_slot)
        return k

    def _loop_on_static_buffers(self, plan, guidance_scale, ts_rows, use_controlnet=False, refiner_start_step=None,
                                inpaint=None, blend=None, guided=True):
        """The whole N-step loop on static device buffers (no host-side tensor arguments): what the loop graph
        captures.  Prologue, once per prompt: cross-attention K/V of all blocks from the text states, the
        time-embedding biases of all ResNet blocks for ALL timesteps (`ts_rows`: each step's timestep repeated per
        batch row, a device tensor made outside the capture), the first UNet input.  Per step: the UNet launch
        sequence and ONE fused kernel for guidance + scheduler update, which also writes the next step's UNet
        input (fp16 NHWC, both CFG halves: pipeline.py:502 np.concatenate([latents] * 2)) -- no fill / copy /
        layout kernels in between.  ``inpaint`` ("blend" / "unet9", see ``_inpaint_kind``): "blend" runs the step
        kernel's blend with ``blend[i]`` = (a, b) of step i; "unet9" writes the five conditioning channels (mask,
        masked image latents) into both halves of the first UNet input, which the step kernel never overwrites.
        ``guided=False``: the guidance-free loop: every launch (K/V prologue, time table, UNet, ControlNets, step)
        sees only the N prompt rows [0, N) of the static buffers; ``ts_rows`` holds N entries per step."""
        n = self.images_per_call
        rows = self.unet.batch if guided else n
        rs = len(plan) if refiner_start_step is None else max(0, min(len(plan), refiner_start_step))
        # which UNet runs each step: the SDXL refiner takes over at refiner_start_step with its own conditioning
        # (StableDiffusionXLPipeline.swift:205-225); each model gets its per-prompt prologue and its own time table
        models = [self.unet if i < rs else self.unet_refiner for i in range(len(plan))]
        # use_controlnet: False, or per step the tuple of ControlNets that run (controlnet_keep)
        keep = use_controlnet if isinstance(use_controlnet, (list, tuple)) else [None] * len(plan)
        self._hist.zero_()
        tables = {}
        for m, lo, hi in ((self.unet, 0, rs), (self.unet_refiner, rs, len(plan))):
            if hi > lo:
                m.prepare_prompt(rows)
                tables[id(m)] = (m.time_table(ts_rows[lo * rows: hi * rows], rows), lo)
        first = models[0]
        x_in = self._latents
        if inpaint == "unet9":
            x_in = self._inpaint_bufs["unet_in"]
            x_in[:, :self.latent_channels].copy_(self._latents)
        L.nchw_to_nhwc(x_in, c_pad=first.engine.in_pad, out=first._x_nhwc[:n])
        if guided:
            L.nchw_to_nhwc(x_in, c_pad=first.engine.in_pad, out=first._x_nhwc[n:])
        if use_controlnet:
            self.prepare_controlnets(ts_rows, rows)
        for i, st in enumerate(plan):
            u = models[i]
            table, lo = tables[id(u)]
            u._run_core(table[i - lo], self.controlnet_residuals(i, rows=rows, nets=keep[i]) if use_controlnet else None,
                        rows)
            k = self._coeffs(st, guidance_scale)
            k.noise_pred_nhwc = 1
            nxt = models[i + 1] if i + 1 < len(plan) else u
            self._step(st, k, u._out_nhwc[:rows], unet_in=nxt._x_nhwc, blend=blend[i] if blend else None,
                       guided=guided)

    def _step(self, st, k, noise_pred, unet_in=None, blend=None, guided=True):
        """One fused guidance + scheduler update of the loop state, with the step's noise when the plan has some and
        the inpainting blend with ``blend`` = (a, b) when given.  ``guided=False``: ``noise_pred`` holds one
        prediction per image and the step kernel's guidance-free mode runs."""
        noised = st.noise_offset >= 0
        if not guided:
            b = self._inpaint_bufs
            L.scheduler_step_guidance_free(
                noise_pred, self._latents, k, st.noise_scale if noised else 0.0, self._noise_key if noised else None,
                self._noise_base + st.noise_offset if noised else 0,
                blend=(b["mask"], b["image_latents"], b["noise"], blend[0], blend[1]) if blend is not None else None,
                hist=self._hist, denoised=self._denoised, unet_in=unet_in)
        elif blend is not None:
            b = self._inpaint_bufs
            L.cfg_scheduler_step_blend(noise_pred, self._latents, k, b["mask"], b["image_latents"], b["noise"],
                                       blend[0], blend[1], st.noise_scale if noised else 0.0,
                                       self._noise_key if noised else None,
                                       self._noise_base + st.noise_offset if noised else 0, hist=self._hist,
                                       denoised=self._denoised, unet_in=unet_in)
        elif st.noise_offset >= 0:
            L.cfg_scheduler_step_noised(noise_pred, self._latents, k, st.noise_scale, self._noise_key,
                                        self._noise_base + st.noise_offset, hist=self._hist, denoised=self._denoised,
                                        unet_in=unet_in)
        else:
            L.cfg_scheduler_step(noise_pred, self._latents, k, hist=self._hist, denoised=self._denoised,
                                 unet_in=unet_in)

    def _inpaint_kind(self, inpainting, start_step=0, controlnet=False, refiner=False):
        """None (no inpainting), "blend" (a 4-channel UNet: the step kernel blends the noised image back in) or
        "unet9" (a 9-channel inpainting UNet: mask and masked image latents are UNet input channels).  Raises a
        ValueError naming any combination the inpainting loop does not support."""
        cin = self.unet.in_channels
        if not inpainting:
            if cin == 9:
                raise ValueError("the UNet is an inpainting UNet (in_channels=9): pass mask_image and starting_image")
            return None
        if cin not in (4, 9):
            raise ValueError(f"inpainting runs UNets with in_channels 4 or 9, this one has in_channels={cin}")
        if self.unet.engine.xl:
            raise ValueError("inpainting is not supported for SDXL (text_time) UNets")
        if refiner or self.unet_refiner is not None:
            raise ValueError("inpainting is not supported with the SDXL refiner")
        if controlnet or self.controlnet:
            raise ValueError("inpainting is not supported with ControlNet")
        if start_step and self.scheduler_name not in INPAINT_STRENGTH_SCHEDULERS:
            raise ValueError(f"inpainting at strength < 1 is not supported for the {self.scheduler_name} scheduler "
                             f"(only {INPAINT_STRENGTH_SCHEDULERS})")
        return "unet9" if cin == 9 else "blend"

    def _set_inpaint_buffers(self, kind, inp):
        """Copy one call's mask and image latents into the static buffers the loop (graph) reads."""
        n, c, h, w = self._latents.shape
        if self._inpaint_bufs is None:
            zeros = lambda *s: torch.zeros(*s, dtype=torch.float32, device=self.device)  # noqa: E731
            self._inpaint_bufs = {"mask": zeros(n, 1, h, w), "image_latents": zeros(n, c, h, w),
                                  "noise": zeros(n, c, h, w), "unet_in": zeros(n, self.unet.in_channels, h, w)}
        b = self._inpaint_bufs
        as_dev = lambda v, shape: torch.as_tensor(v, dtype=torch.float32).to(self.device).reshape(shape)  # noqa: E731
        mask = as_dev(inp.mask, (n, 1, h, w))
        b["mask"].copy_(mask)
        if kind == "blend":
            b["image_latents"].copy_(as_dev(inp.image_latents, (n, c, h, w)))
            b["noise"].copy_(as_dev(inp.noise, (n, c, h, w)))
        else:
            b["unet_in"][:, c:c + 1].copy_(mask)
            b["unet_in"][:, c + 1:].copy_(as_dev(inp.masked_image_latents, (n, self.unet.in_channels - c - 1, h, w)))

    def set_control_scales(self, scales, keep=None):
        """Write the conditioning scales (one float per net) into the device arrays the loop reads: one per set of
        nets in ``keep`` (per-step tuples, controlnet_keep), allocated on first use, and the set of all nets."""
        sets = {self._all_nets} | set(keep or ())
        for nets in sets:
            if not nets:
                continue
            buf = self._control_scale_bufs.get(nets)
            if buf is None:
                buf = self._control_scale_bufs[nets] = torch.empty(len(nets), dtype=torch.float32, device=self.device)
            buf.copy_(torch.tensor([scales[k] for k in nets], dtype=torch.float32))

    def set_control_conditions(self, controlnet_cond):
        """Copy the conditioning images (each (2B, 3, H, W)) into the ControlNets' static input buffers."""
        for module, cond in zip(self.controlnet, controlnet_cond):
            cond = torch.as_tensor(cond)
            module._cond[:cond.shape[0]].copy_(cond)

    def prepare_controlnets(self, ts_rows, rows=None):
        """Device-loop prologue of every ControlNet: text states, the embedding of its conditioning image (static
        buffer `_cond`), time-embedding table (of the first ``rows`` images: the guidance-free loop)."""
        for module in self.controlnet:
            module._ctx.copy_(self.unet._ctx)
            if module.engine.xl:  # the add-embedding rows the UNet gets (the negative pooled embedding on uncond rows)
                module._time_ids.copy_(self.unet._time_ids)
                module._text_embeds.copy_(self.unet._text_embeds)
            module.prepare_prompt(ts_rows, rows)

    def controlnet_residuals(self, step, _temb=None, rows=None, nets=None):
        """pipeline.py:259-284 inside the device loop: the ControlNets ``nets`` (indices; default all) see the UNet's
        input.  -> ControlResiduals for the UNet, which scales and sums them as it injects them, or None when ``nets``
        is empty."""
        nets = self._all_nets if nets is None else tuple(nets)
        if not nets:
            return None
        x = self.unet._x_nhwc if rows is None else self.unet._x_nhwc[:rows]
        return ControlResiduals([self.controlnet[k].run_core(x, step) for k in nets], self._control_scale_bufs[nets])

    def _ts_rows(self, plan, rows=None):
        return torch.tensor([float(st.timestep) for st in plan for _ in range(rows or self.unet.batch)],
                            dtype=torch.float32, device=self.device)

    def _loop_graph_for(self, key, plan, guidance_scale, use_controlnet=False, refiner_start_step=None, inpaint=None,
                        blend=None, guided=True):
        g = self._loop_graphs.get(key)
        if g is None:
            keep = self._latents.clone()
            rows = self.unet.batch if guided else self.images_per_call
            ts_rows = self._ts_rows(plan, rows)
            s = torch.cuda.Stream(device=self.device)  # eager warm-up off the capture: workspaces, weight tiling
            s.wait_stream(torch.cuda.current_stream())
            with torch.cuda.stream(s):
                # every ControlNet runs in the warm-up step, whichever steps it is kept at
                self._loop_on_static_buffers(plan[:1], guidance_scale, ts_rows[:rows],
                                             [self._all_nets] if use_controlnet else False,
                                             inpaint=inpaint, blend=blend[:1] if blend else None, guided=guided)
                if refiner_start_step is not None and refiner_start_step < len(plan):  # warm the refiner's kernels too
                    self._loop_on_static_buffers(plan[-1:], guidance_scale, ts_rows[-rows:], use_controlnet, 0)
            torch.cuda.current_stream().wait_stream(s)
            torch.cuda.synchronize()
            self._latents.copy_(keep)
            g = torch.cuda.CUDAGraph()
            with torch.cuda.graph(g):
                self._loop_on_static_buffers(plan, guidance_scale, ts_rows, use_controlnet, refiner_start_step,
                                             inpaint, blend, guided)
            g._b200sd_keep = ts_rows
            self._latents.copy_(keep)  # capture does not execute, but keep the contract obvious
            if len(self._loop_graphs) >= 4:
                self._loop_graphs.pop(next(iter(self._loop_graphs)))
            self._loop_graphs[key] = g
        return g

    def denoise(self, text_embeddings, latents, num_inference_steps, guidance_scale, callback=None,
                callback_steps=1, time_ids=None, text_embeds=None, return_denoised=False, record=None,
                controlnet_cond=None, start_step=0, refiner=None, refiner_start=0.8, noise_key=None, noise_offset=0,
                inpaint=None, controlnet_conditioning_scale=1.0, control_guidance_start=0.0, control_guidance_end=1.0):
        """Runs the N-step loop (from ``start_step``: image-to-image) entirely on the device.  ``text_embeddings`` (2B, D, 1, S) and ``latents``
        (B, C, h, w) may be numpy (copied once, before the loop) or CUDA tensors.  ``record`` (a list) receives
        (timestep, noise_pred, latents_after_step) clones per step -- a debugging / testing aid.  Without
        callback / record / ControlNet the whole loop replays as ONE CUDA graph (SURVEY 8f N1): the scheduler
        history lives on the device and no host synchronisation happens between the first and the last step.
        Latents in and out (and those given to ``record`` / ``callback``) are x-space; the Euler / LMS samplers loop on
        x / sqrt(sigma^2 + 1), so their latents are divided once before the loop and multiplied back off the hot path.
        ``noise_key`` / ``noise_offset`` (ancestral samplers): step j adds the Philox normals of
        ``NvRandomSource(noise_key)``'s draw number ``noise_offset + j``; without a key one ``np.random.randint(2**32)``
        is drawn.
        ``inpaint`` (``InpaintInputs``): the latent mask and image latents of an inpainting call (``__call__`` with
        ``mask_image``); required for a 9-channel UNet.  They are copied into static buffers before the loop, so the
        loop graph depends on the inpainting kind only, never on the mask or the images.
        ``controlnet_conditioning_scale`` / ``control_guidance_start`` / ``control_guidance_end``: a float or one per
        ControlNet (controlnet_arguments); net k runs at the steps controlnet_keep gives and is not launched at the
        others.  The loop graph is keyed by those per-step sets of nets, not by the scales, which it reads on the
        device.

        Without classifier-free guidance (``do_classifier_free_guidance``: guidance_scale <= 1, or a guidance-embedding
        UNet) the loop runs guidance-free: the UNet (still built at batch 2B) and the ControlNets run on B rows only.
        ``text_embeddings``, ``time_ids`` and ``text_embeds`` may then have B rows, or 2B in the uncond-first layout,
        whose second (prompt) half is taken.  A guidance-embedding UNet is conditioned on
        ``unet.guidance_scale_embedding(guidance_scale)``."""
        sched = S.make_scheduler(self.scheduler_name, num_inference_steps, **self.scheduler_kwargs)
        plan = list(sched.plan(start=start_step)) if start_step else list(sched.plan())
        n = self.images_per_call
        guided = self.do_classifier_free_guidance(guidance_scale)
        rows = self.unet.batch if guided else n
        if refiner is not None and not guided:
            raise ValueError("the SDXL refiner hand-off runs with classifier-free guidance only (guidance_scale > 1)")
        kind = self._inpaint_kind(inpaint is not None, start_step, bool(controlnet_cond), refiner is not None)
        blend = None
        if kind is not None:
            self._set_inpaint_buffers(kind, inpaint)
            if kind == "blend":
                blend = sched.blend_coeffs(start_step)
        if guided:
            self._ctx.copy_(torch.as_tensor(text_embeddings), non_blocking=True)
        else:
            text_embeddings = torch.as_tensor(text_embeddings)
            if text_embeddings.shape[0] not in (n, 2 * n):
                raise ValueError(f"text_embeddings has {text_embeddings.shape[0]} rows, expected {n} or {2 * n}")
            self._ctx[:n].copy_(text_embeddings[-n:], non_blocking=True)
            if time_ids is not None:
                time_ids = torch.as_tensor(time_ids).reshape(-1, self.unet._time_ids.shape[1])[-n:]
            if text_embeds is not None:
                text_embeds = torch.as_tensor(text_embeds)[-n:]
        if self.unet.engine.time_cond_dim:
            from .unet import guidance_scale_embedding
            self.unet._cond[:n].copy_(guidance_scale_embedding(guidance_scale, self.unet.engine.time_cond_dim, n))
        self._latents.copy_(torch.as_tensor(latents), non_blocking=True)
        if sched.input_scale(0) != 1.0:
            self._latents.div_(sched.input_scale(0))
        if any(st.noise_offset >= 0 for st in plan):
            key = int(np.random.randint(2 ** 32) if noise_key is None else noise_key) & 0xFFFFFFFF
            self._noise_key.fill_(key - (1 << 32) if key >= 1 << 31 else key)  # the key's bits as int32
        self._noise_base = int(noise_offset)

        def x_space(i):  # latents after i steps, in x-space
            s = sched.input_scale(i)
            return self._latents if s == 1.0 else self._latents * s
        keep = None
        if controlnet_cond:
            if len(controlnet_cond) != len(self.controlnet):
                raise ValueError(f"{len(controlnet_cond)} conditioning images for {len(self.controlnet)} ControlNet(s)")
            scales, starts, ends = controlnet_arguments(len(self.controlnet), controlnet_conditioning_scale,
                                                        control_guidance_start, control_guidance_end)
            keep = controlnet_keep(len(plan), starts, ends)
            self.set_control_scales(scales, keep)
            controlnet_cond = [torch.as_tensor(c).to(self.device, torch.float16) for c in controlnet_cond]
            if not guided:  # the condition images of the B prompt rows (prepare_control_cond doubles them)
                controlnet_cond = [c[-n:] for c in controlnet_cond]
        elif self.unet._res:
            # a UNet built with additional_residual inputs but called without conditions: the static residual buffers
            # would still hold the previous ControlNet call's last step (the reference cannot run this combination)
            for buf in self.unet._res:
                buf.zero_()
        if self.loop_graph and callback is None and record is None:
            u = self.unet
            u._ctx.copy_(self._ctx)
            if u.engine.xl:
                u._time_ids[:rows].copy_(torch.as_tensor(time_ids).reshape(rows, -1))
                u._text_embeds[:rows].copy_(torch.as_tensor(text_embeds))
            if controlnet_cond:
                self.set_control_conditions(controlnet_cond)
            rstep = None
            if refiner is not None:
                if self.unet_refiner is None:
                    raise ValueError("refiner inputs were given but the pipeline has no unet_refiner")
                r = self.unet_refiner
                r._ctx.copy_(torch.as_tensor(refiner["encoder_hidden_states"]))
                r._time_ids.copy_(torch.as_tensor(refiner["time_ids"]).reshape(r._time_ids.shape))
                r._text_embeds.copy_(torch.as_tensor(refiner["text_embeds"]))
                rstep = int(np.float32(len(plan)) * np.float32(refiner_start))  # Int(Float(timeSteps.count) * refinerStart)
            key = (self.scheduler_name, int(num_inference_steps), float(guidance_scale), int(start_step),
                   tuple(keep) if keep else None, tuple(sorted(self.scheduler_kwargs.items())), rstep, self._noise_base,
                   guided, kind)
            self._loop_graph_for(key, plan, guidance_scale, keep or False, rstep, kind, blend, guided).replay()
            return self._denoised if return_denoised else self._latents
        if refiner is not None:
            raise ValueError("the refiner hand-off runs in the device loop only (no callback / record)")
        self._hist.zero_()
        k = L.StepCoeffs()
        for i, st in enumerate(plan):
            self._t.fill_(float(st.timestep))
            x_in = self._latents
            if kind == "unet9":  # cat([latents, mask, masked_image_latents], 1), the same conditioning every step
                x_in = self._inpaint_bufs["unet_in"]
                x_in[:, :self.latent_channels].copy_(self._latents)
            sample = torch.cat([x_in, x_in], 0) if guided else x_in  # pipeline.py:502
            residuals = None
            if controlnet_cond:  # pipeline.py:515-529
                residuals = self.run_controlnet(sample, self._t[:rows], self._ctx[:rows], controlnet_cond, keep[i],
                                                time_ids, text_embeds)
                if residuals is None:  # no net runs at this step: nothing is injected
                    for buf in self.unet._res:
                        buf[:rows].zero_()
            noise_pred = self.unet.forward_device(sample, self._t[:rows], self._ctx[:rows], time_ids, text_embeds,
                                                  residuals, self.unet._cond[:rows] if self.unet._cond is not None
                                                  else None)
            self._coeffs(st, guidance_scale, k)
            if record is not None:
                eps_copy = noise_pred.clone()
            self._step(st, k, noise_pred, blend=blend[i] if blend else None, guided=guided)
            if record is not None:
                record.append((st.timestep, eps_copy, x_space(i + 1).clone()))
            if callback is not None and i % callback_steps == 0:
                callback(i, st.timestep, x_space(i + 1))
        return self._denoised if return_denoised else self._latents

    def calibrate_unet(self, prompts, num_inference_steps=50, guidance_scale=7.5, seed=0, linear=False):
        """W8A8 calibration: runs the denoising loop eagerly with the fp16 UNet once per prompt (seed, seed + 1, ...)
        and records max |x| at the input of every convolution the engine can quantize, over every UNet call (all
        steps, both classifier-free-guidance halves).  linear: the transformer linears too (the recipe's linear
        section).  Returns the ``quantization.W8A8Recipe`` with s_a = amax / 127 for all of them;
        ``from_pretrained(..., unet_quantization=recipe)`` (or ``recipe.save(path)``) applies it."""
        from .quantization import W8A8Recipe, quantizable_linear_layers
        if isinstance(prompts, str):
            prompts = [prompts]
        u = self.unet
        eng = u.engine
        slots = eng.set_calibration(True, linear=linear)
        graphed, u.use_cuda_graph = u.use_cuda_graph, False  # the probes must not enter a captured graph
        try:
            for i, p in enumerate(prompts):
                # a callback keeps denoise() on the step-by-step path, where every UNet call runs eagerly
                self(p, height=self.height, width=self.width, num_inference_steps=num_inference_steps,
                     guidance_scale=guidance_scale, seed=seed + i, output_type="np", callback=lambda *a: None)
            torch.cuda.synchronize(self.device)
        finally:
            u.use_cuda_graph = graphed
            eng.set_calibration(False)
        amax = {n: float(t.item()) for n, t in slots.items()}
        lin = quantizable_linear_layers(eng.cfg)
        return W8A8Recipe.from_amax({n: v for n, v in amax.items() if n not in lin}, eng.cfg,
                                    {n: v for n, v in amax.items() if n in lin})

    def decode_latents(self, latents, want_u8=False):
        """pipeline.py:313-320 on the device: z / scaling -> decoder -> clip(x/2+0.5, 0, 1) -> NHWC fp32 (and, with
        ``want_u8``, numpy_to_pil's u8 pixels round(255 x))."""
        eng = self.vae_decoder.engine
        self.vae_decoder._z.copy_(latents)
        self.vae_decoder._z.mul_(1.0 / eng.scaling)
        img = eng.forward(self.vae_decoder._z)
        return L.image_postprocess(img, c=eng.out_ch, want_u8=want_u8)

    def decode_and_check(self, latents):
        """Decode, then pipeline.py:286-311 on the device: CLIP preprocessing of the u8 pixels, the vision tower,
        concept scoring, flagged images zeroed -- and one copy of images and flags to the host at the end.  Differs
        from the reference by design in two ways: the returned images keep the pipeline's fp32 values (the reference
        casts them to fp16 for the Core ML call and returns that cast), and the flags are a List[bool], the type
        StableDiffusionPipelineOutput declares (the reference passes its raw (B, 1, 1, 1) array through).
        -> (images float32 NHWC numpy, nsfw_content_detected or None without a checker)."""
        if self.safety_checker is None:
            return self.decode_latents(latents).cpu().numpy(), None
        image, image_u8 = self.decode_latents(latents, want_u8=True)
        flags, _ = self.safety_checker.check(image, image_u8)
        image, flags = image.cpu().numpy(), flags.cpu().numpy()
        return image, [bool(f) for f in flags]

    # ---------------------------------------------------------------- public API
    def __call__(self, prompt, height=512, width=512, num_inference_steps=50, guidance_scale=7.5,
                 negative_prompt=None, num_images_per_prompt=1, eta=0.0, latents=None, output_type="pil",
                 return_dict=True, callback=None, callback_steps=1, controlnet_cond=None,
                 original_size: Optional[Tuple[int, int]] = None, crops_coords_top_left: Tuple[int, int] = (0, 0),
                 target_size: Optional[Tuple[int, int]] = None, unet_batch_one=False, prompt_embeds=None,
                 starting_image=None, strength=None, seed=None, rng="numpy", refiner_start=0.8, aesthetic_score=6.0,
                 negative_aesthetic_score=2.5, mask_image=None, controlnet_conditioning_scale=1.0,
                 control_guidance_start=0.0, control_guidance_end=1.0, guess_mode=False, **kwargs):
        """``starting_image`` ((B, 3, H, W) in [-1, 1], the vae_encoder input) + ``strength`` (default 0.5) select the
        Swift pipeline's image-to-image mode (StableDiffusionPipeline.swift:250-262, 361-378): the encoded image is
        noised to timestep ``timeSteps[startStep]`` and only the remaining steps run.

        ``mask_image`` ((B | 1, 1, H, W) or (H, W) in [0, 1], 1 = repaint) with ``starting_image`` inpaints, as diffusers
        0.30.2's ``StableDiffusionInpaintPipeline`` (``strength`` default 1.0; < 1 for DDIM and DPM-Solver++ only, start
        step ``get_timesteps``'s).  A 9-channel inpainting UNet reads cat([latents, mask, masked image latents]); a
        4-channel UNet keeps the unmasked region by blending the noised image latents back in after every step, so
        the unmasked latents end exactly on the image latents.  Draws from the global numpy stream, after the latent
        noise: the encoder noise of the full image (4-channel UNet, or strength < 1), then that of the masked image
        (9-channel UNet).

        ControlNet (``controlnet_cond``: one (3, H, W) image per net), as diffusers' ControlNet pipelines:
        ``controlnet_conditioning_scale`` multiplies each net's residuals (a float or one per net; SDXL ControlNets are
        usually run at 0.5), and net k runs only at the steps inside its window [``control_guidance_start``,
        ``control_guidance_end``] (fractions of the executed steps).  ``guess_mode`` is not implemented."""
        self.check_inputs(prompt, height, width, callback_steps)
        if guess_mode:
            raise ValueError("guess_mode=True is not implemented")
        height = height or self.height
        width = width or self.width
        if (height, width) != (self.height, self.width):
            raise ValueError(f"this pipeline instance was built for {self.height}x{self.width} images")
        if eta != 0.0:
            raise ValueError("only eta = 0 (deterministic DDIM) is implemented")
        if controlnet_cond and not self.controlnet:
            raise ValueError("Conditions for controlnet are given but the pipeline has no controlnet modules")
        if controlnet_cond:
            controlnet_arguments(len(self.controlnet), controlnet_conditioning_scale, control_guidance_start,
                                 control_guidance_end)
        prompts = [prompt] if isinstance(prompt, str) else list(prompt)
        prompts = [p for p in prompts for _ in range(num_images_per_prompt)]
        if len(prompts) != self.images_per_call:
            raise ValueError(f"this pipeline instance generates {self.images_per_call} image(s) per call, "
                             f"got {len(prompts)} prompt(s)")
        do_cfg = self.do_classifier_free_guidance(guidance_scale)  # pipeline.py:443, and no guidance embedding
        if self.scheduler_name == "LCM":
            for name, v in (("mask_image", mask_image), ("starting_image", starting_image)):
                if v is not None:
                    raise ValueError(f"{name} is not supported with the LCM scheduler (its strength changes the "
                                     f"timesteps themselves)")
        xl_pooled = None
        if prompt_embeds is not None:
            text_embeddings = prompt_embeds
        elif self.xl and self.text_encoder_2 is not None:
            text_embeddings, xl_pooled = self._encode_prompt_xl(prompts, do_cfg, negative_prompt,
                                                                negative_prompt_2=kwargs.get("negative_prompt_2"))
        else:
            text_embeddings = self._encode_prompt(prompts, do_cfg, negative_prompt)
        time_ids = text_embeds = None
        if self.xl:
            original_size = original_size or (height, width)
            target_size = target_size or (height, width)
            ids = list(original_size) + list(crops_coords_top_left) + list(target_size)
            time_ids = torch.tensor([ids] * (2 * self.images_per_call), dtype=torch.float32, device=self.device)
            text_embeds = kwargs.get("pooled_prompt_embeds")
            if text_embeds is None and xl_pooled is not None:
                text_embeds = torch.as_tensor(xl_pooled, dtype=torch.float32, device=self.device)
            if text_embeds is None:
                text_embeds = torch.zeros(2 * self.images_per_call, 1280, device=self.device)
        sched = S.make_scheduler(self.scheduler_name, num_inference_steps, **self.scheduler_kwargs)
        inpaint_kind, start_step = None, 0
        if mask_image is not None or self.unet.in_channels == 9:
            if mask_image is not None and starting_image is None:
                raise ValueError("mask_image needs a starting_image (the image to inpaint)")
            strength = 1.0 if strength is None else float(strength)
            if not 0.0 < strength <= 1.0:
                raise ValueError(f"inpainting strength must be in (0, 1], got {strength}")
            start_step = sched.inpaint_start_step(strength)
            if start_step >= num_inference_steps:
                raise ValueError(f"strength {strength} leaves no denoising steps")
            inpaint_kind = self._inpaint_kind(mask_image is not None, start_step, bool(controlnet_cond))
            if self.vae_encoder is None:
                raise ValueError("inpainting needs a vae_encoder (with_vae_encoder=True)")
        elif starting_image is not None and self.scheduler_name in S.SIGMA_SCHEDULERS:
            raise ValueError(f"image-to-image is not implemented for the {self.scheduler_name} scheduler")
        init_sigma = sched.init_noise_sigma
        if inpaint_kind is None:
            lat = self.prepare_latents(len(prompts), self.latent_channels, height, width, latents, seed=seed, rng=rng,
                                       init_noise_sigma=init_sigma)
        else:
            # diffusers keeps the unscaled noise z: the blend and the strength < 1 start noise both read it
            noise = self.prepare_latents(len(prompts), self.latent_channels, height, width, latents, seed=seed, rng=rng)
            lat = noise * init_sigma
        # ancestral step noise: keyed by the seed, continuing the latents' Philox stream with the nvidia source; without
        # a seed, denoise() draws the key from the global numpy stream right after the latents
        noise_key, noise_offset = None, 0
        if seed is not None:
            noise_key = seed
            noise_offset = len(prompts) if rng in ("nvidia", "nvidiaRNG") else 0
        inpaint = None
        if inpaint_kind is not None:
            mask_img, masked = prepare_mask_and_masked_image(starting_image, mask_image)
            enc_dtype = self.vae_encoder.expected_inputs["x"]["dtype"]
            scaling = self.vae_decoder.engine.scaling
            x0 = masked_lat = None
            if inpaint_kind == "blend" or start_step:
                enc_noise = np.random.randn(*lat.shape).astype(np.float32)
                x0 = self.vae_encoder.encode(np.asarray(starting_image, dtype=enc_dtype), enc_noise,
                                             scaling).numpy().astype(np.float32)
            if inpaint_kind == "unet9":
                enc_noise = np.random.randn(*lat.shape).astype(np.float32)
                masked_lat = self.vae_encoder.encode(masked.astype(enc_dtype), enc_noise, scaling).numpy().astype(np.float32)
            if start_step:
                a, b = sched.noise_coeffs(start_step)  # add_noise(image_latents, noise, timesteps[t_start])
                lat = np.float32(a) * x0 + np.float32(b) * noise
            inpaint = InpaintInputs(latent_mask(mask_img, self.vae_scale_factor), x0, noise, masked_lat)
        elif starting_image is not None:
            strength = 0.5 if strength is None else strength
            if self.vae_encoder is None:
                raise ValueError("a starting image was provided but the pipeline has no vae_encoder")
            sched = S.make_scheduler(self.scheduler_name, num_inference_steps, **self.scheduler_kwargs)
            start_step = sched.start_step(strength)
            if start_step >= num_inference_steps:
                raise ValueError(f"strength {strength} leaves no denoising steps")
            # same draw order as the Swift pipeline: the noise samples first (above), then the encoder's noise
            enc_noise = np.random.randn(*lat.shape).astype(np.float32)
            x0 = self.vae_encoder.encode(np.asarray(starting_image, dtype=self.vae_encoder.expected_inputs["x"]["dtype"]),
                                         enc_noise, self.vae_decoder.engine.scaling).numpy()
            lat = sched.add_noise(x0.astype(np.float32), lat, strength)
        if controlnet_cond:  # pipeline.py:488-494
            controlnet_cond = self.prepare_control_cond(controlnet_cond, do_cfg, len(prompts), 1)
        refiner = None
        if self.unet_refiner is not None:
            # refiner conditioning (StableDiffusionXLPipeline.swift:314-345): the second encoder's embeddings only, its
            # pooled output, geometry = (original size, crop, aesthetic score) with the negative score on the uncond row
            r_emb = kwargs.get("refiner_prompt_embeds")
            r_pool = kwargs.get("refiner_pooled_prompt_embeds")
            if r_emb is None:
                if self.text_encoder_2 is None:
                    raise ValueError("the refiner needs text_encoder_2 or refiner_prompt_embeds / refiner_pooled_prompt_embeds")
                r_emb, r_pool = self._encode_prompt_xl(prompts, do_cfg, negative_prompt, only_second=True,
                                                       negative_prompt_2=kwargs.get("negative_prompt_2"))
            osz, crop = list(original_size or (height, width)), list(crops_coords_top_left)
            rows = [osz + crop + [negative_aesthetic_score]] * self.images_per_call + \
                   [osz + crop + [aesthetic_score]] * self.images_per_call
            refiner = {"encoder_hidden_states": r_emb, "text_embeds": torch.as_tensor(np.asarray(r_pool), dtype=torch.float32),
                       "time_ids": torch.tensor(rows, dtype=torch.float32)}
        final = self.denoise(text_embeddings, lat, num_inference_steps, guidance_scale, callback, callback_steps,
                             time_ids, text_embeds, controlnet_cond=controlnet_cond or None, start_step=start_step,
                             refiner=refiner, refiner_start=refiner_start, noise_key=noise_key,
                             noise_offset=noise_offset, inpaint=inpaint,
                             controlnet_conditioning_scale=controlnet_conditioning_scale,
                             control_guidance_start=control_guidance_start, control_guidance_end=control_guidance_end)
        image, has_nsfw = self.decode_and_check(final)  # the only device->host copies of the result
        if output_type == "pil":
            image = self.numpy_to_pil(image)
        if not return_dict:
            return (image, has_nsfw)
        return StableDiffusionPipelineOutput(images=image, nsfw_content_detected=has_nsfw)

    def generate(self, prompt, num_inference_steps=50, guidance_scale=7.5, **kwargs):
        """Alias named in BASELINE.json's north_star."""
        return self(prompt, num_inference_steps=num_inference_steps, guidance_scale=guidance_scale, **kwargs)
