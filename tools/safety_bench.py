"""Time of the safety checker, alone and inside the SD-1.5 pipeline.

    python tools/safety_bench.py [--iters 20] [--rounds 5]

1. The checker stage alone (``SafetyCheckerEngine.check``: CLIP preprocessing of 512x512 u8 images, the ViT-L/14
   tower, concept scoring, filter), random-init SD-1.x checker weights, at batch 1 and 8: CUDA events around
   ``--iters`` calls after a warm-up, ms per call.
2. End to end: ``B200StableDiffusionPipeline.__call__`` of SD-1.5 (random init) at 512x512, one image, 20 DDIM steps,
   CFG 7.5, output_type "np", with and without the checker, alternated ``--rounds`` times; host clock around each
   call (the call ends in a device-to-host copy), median seconds per call.
Prints one JSON line with the card name and power limit."""
import argparse
import json
import os
import statistics
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import torch  # noqa: E402


def power_limit_w(index):
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader,nounits", "-i", str(index)],
                             stdout=subprocess.PIPE, stderr=subprocess.DEVNULL, text=True, timeout=10).stdout.strip()
        return float(out)
    except Exception:
        return None


def checker_ms(eng, batch, iters, dev):
    g = torch.Generator(device=dev).manual_seed(batch)
    u8 = torch.randint(0, 256, (batch, 512, 512, 3), generator=g, device=dev, dtype=torch.uint8)
    img = u8.float() / 255
    for _ in range(3):
        eng.check(img, u8)
    torch.cuda.synchronize()
    t0, t1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    t0.record()
    for _ in range(iters):
        eng.check(img, u8)
    t1.record()
    torch.cuda.synchronize()
    return t0.elapsed_time(t1) / iters


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--rounds", type=int, default=5)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        print(json.dumps({"error": "no CUDA device: the safety checker runs on the GPU only"}))
        sys.exit(1)
    from b200sd import config as C
    from b200sd.pipeline import B200StableDiffusionPipeline as P

    dev = torch.device("cuda:0")
    pipe = P.from_random_init("sd15", images_per_call=1, seed=0, safety_checker_cfg=C.SD_SAFETY_CHECKER)
    eng = pipe.safety_checker
    res = {"checker_ms_b1": checker_ms(eng, 1, args.iters, dev), "checker_ms_b8": checker_ms(eng, 8, args.iters, dev)}
    run = dict(num_inference_steps=20, guidance_scale=7.5, output_type="np", seed=1)
    pipe("a photo", **run)
    times = {"with": [], "without": []}
    for _ in range(args.rounds):
        for mode in ("without", "with"):
            pipe.safety_checker = eng if mode == "with" else None
            torch.cuda.synchronize()
            t = time.perf_counter()
            pipe("a photo", **run)
            times[mode].append(time.perf_counter() - t)
    res.update({f"e2e_s_{k}_checker": statistics.median(v) for k, v in times.items()})
    res.update({"e2e_rounds": args.rounds, "card": torch.cuda.get_device_name(dev), "power_limit_w": power_limit_w(0)})
    print(json.dumps(res), flush=True)


if __name__ == "__main__":
    main()
