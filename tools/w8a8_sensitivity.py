"""Per-layer W8A8 sensitivity (the reference's activation_quantization.py step 2) on this engine: for every convolution
the engine can quantize, quantize that layer alone, run the denoising loop to the final latents for each prompt and take
the mean PSNR against the fp16 UNet's latents (the formula of oracle.restated.compute_psnr).  Writes the reference's
JSON format, {"conv": {layer: psnr}, "einsum": {}, "model_version": ...}, which quantization.select_from_sensitivity
reads with a conv_psnr threshold.  Prompts come from the user.  SD 1.x / 2.x pipelines (one text encoder).
--linear: the transformer linears too, under the reference's names in the same "conv" section (its UNet runs them as 1x1
convolutions); an attn1 to_q / to_k / to_v triple is one launch here, so its three entries get the PSNR of quantizing the
triple.

    python tools/w8a8_sensitivity.py --model-dir DIR --prompt "..." --prompt "..." --steps 20 --out sens.json
    python tools/w8a8_sensitivity.py --random-init sd21-base --prompt "..." --out sens.json   (random weights)
"""
import argparse
import json
import os
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))


def main():
    ap = argparse.ArgumentParser()
    src = ap.add_mutually_exclusive_group(required=True)
    src.add_argument("--model-dir")
    src.add_argument("--random-init", choices=["sd21-base", "sd15", "tiny"])
    ap.add_argument("--prompt", action="append", required=True)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--guidance-scale", type=float, default=7.5)
    ap.add_argument("--seed", type=int, default=0)
    ap.add_argument("--recipe", help="calibrated W8A8Recipe JSON (default: calibrate on the prompts)")
    ap.add_argument("--layers", nargs="*", help="restrict to these layers")
    ap.add_argument("--linear", action="store_true", help="also the transformer linears (select_from_sensitivity(linear=True))")
    ap.add_argument("--out", required=True)
    args = ap.parse_args()
    from b200sd import checkpoint as K
    from b200sd import config as C
    from b200sd.model import UNetModel
    from b200sd.pipeline import B200StableDiffusionPipeline as P
    from b200sd.quantization import W8A8Recipe, compute_psnr

    if args.model_dir:
        pipe = P.from_pretrained(args.model_dir, load_safety_checker=False)
        cfg = K.read_config(args.model_dir, "unet")
        sd = K.load_component(args.model_dir, "unet", cfg)
        version = os.path.basename(os.path.normpath(args.model_dir))
    else:
        pipe = P.from_random_init(args.random_init, seed=args.seed)
        cfg = {"sd21-base": C.SD21_BASE_UNET, "sd15": C.SD15_UNET, "tiny": C.TINY_UNET}[args.random_init]
        sd = C.random_state_dict(C.unet_param_shapes(cfg), seed=args.seed, dtype=torch.float16)
        version = f"random-init {args.random_init}"
    if pipe.xl:
        raise SystemExit("w8a8_sensitivity: SD 1.x / 2.x pipelines only")
    recipe = W8A8Recipe.load(args.recipe) if args.recipe else pipe.calibrate_unet(
        args.prompt, num_inference_steps=args.steps, guidance_scale=args.guidance_scale, seed=args.seed,
        linear=args.linear)
    u16 = pipe.unet
    rs = np.random.RandomState(args.seed)
    lat = torch.from_numpy(rs.randn(1, 4, u16.h, u16.w).astype(np.float32))
    embs = [pipe._encode_prompt([p], True, None) for p in args.prompt]

    def final_latents(unet):
        pipe.unet = unet
        pipe._loop_graphs = {}
        return [pipe.denoise(e, lat, args.steps, args.guidance_scale).cpu().clone() for e in embs]

    ref = final_latents(u16)
    results = {}
    layers = args.layers or (list(recipe.scales) + (list(recipe.linear_scales) if args.linear else []))
    for layer in layers:
        if layer in results:
            continue
        if layer in recipe.linear_scales:
            block = layer.rsplit(".", 1)[0]
            group = [f"{block}.to_{n}" for n in "qkv"] if block.endswith(".attn1") else [layer]
            sub = recipe.subset([], group)
        else:
            group, sub = [layer], recipe.subset([layer])
        uq = UNetModel(cfg, sd, batch=u16.batch, height=u16.h, width=u16.w, quantization=sub)
        outs = final_latents(uq)
        for n in group:
            results[n] = float(np.mean([compute_psnr(r, o) for r, o in zip(ref, outs)]))
        print(f"{layer}: {results[layer]:.2f} dB", flush=True)
        del uq
        torch.cuda.empty_cache()
    pipe.unet = u16
    with open(args.out, "w") as f:
        json.dump({"conv": results, "einsum": {}, "model_version": version}, f, indent=2)


if __name__ == "__main__":
    main()
