"""Iter/s of the device denoising loop for one model, with the attention kernels' share of a step.

    python tools/model_bench.py --model sd15|sd21-base|sd21 [--reps 3]

The workload is bench.py's: random-init weights, txt2img 512x512 at UNet batch 2 (uncond, cond), 20 DDIM steps, CFG
7.5, the 20 steps (with the per-prompt prologue) captured as one CUDA graph by bench.LoopBench and timed with
bench.timed_replays.  ``sd21`` (SD 2.0 / 2.1 768-v) runs the same UNet at 768x768 (96x96 latents) with 20 DDIM
v-prediction steps.  The attention time is the same loop captured with only the attention class launching
(classes=2).  Prints one JSON line: iter/s, ms per step, attention ms per step, card name, power limit and the median
SM clock while the loop ran."""
import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import torch  # noqa: E402

import bench  # noqa: E402


def power_limit_w(index):
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader,nounits", "-i", str(index)],
                             stdout=subprocess.PIPE, stderr=subprocess.DEVNULL, text=True, timeout=10).stdout.strip()
        return float(out)
    except Exception:
        return None


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n")[0])
    ap.add_argument("--model", choices=("sd15", "sd21-base", "sd21"), default="sd15")
    ap.add_argument("--reps", type=int, default=3, help="replays of the 20-step graph per measurement")
    args = ap.parse_args()

    from b200sd import lib as L
    from b200sd import scheduler as S
    from b200sd.pipeline import B200StableDiffusionPipeline

    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    L.load()
    pipe = B200StableDiffusionPipeline.from_random_init(args.model, images_per_call=1, device=dev, seed=1,
                                                        scheduler="DDIM")
    d_ctx = pipe.unet._ctx.shape[1]
    g = torch.Generator().manual_seed(93)
    pipe.unet._ctx.copy_(torch.cat([torch.zeros(1, d_ctx, 1, 77), torch.randn(1, d_ctx, 1, 77, generator=g)]).half())
    lat0 = torch.randn(1, 4, pipe.unet.h, pipe.unet.w, generator=g).half().float().to(dev)
    loop = bench.LoopBench(pipe, lat0)
    n = bench.N_STEPS_IMG
    loop.plan = S.DDIMScheduler(n, **pipe.scheduler_kwargs).plan()
    pred = pipe.scheduler_kwargs.get("prediction_type", "epsilon")
    full = loop.capture(n)
    attn = loop.capture(n, classes=2)
    sync = torch.cuda.synchronize
    sampler = bench.ClockSampler(0)
    sampler.start()
    ms = bench.timed_replays(full, args.reps, sync) / n
    ms_attn = bench.timed_replays(attn, args.reps, sync) / n
    clocks = sampler.stop()
    workload = f"txt2img {pipe.height}x{pipe.width}, UNet batch 2, 20 DDIM steps ({pred}), CFG 7.5, fp16"
    print(json.dumps({"model": args.model, "workload": workload,
                      "iter_per_s": round(1e3 / ms, 2), "ms_per_step": round(ms, 4),
                      "attention_ms_per_step": round(ms_attn, 4),
                      "launches_per_step": round(loop.launches_per_image / n, 1),
                      "card": torch.cuda.get_device_name(dev), "power_limit_w": power_limit_w(0),
                      "sm_mhz": clocks.get("sm_mhz"), "clock_events": clocks.get("reasons")}), flush=True)


if __name__ == "__main__":
    main()
