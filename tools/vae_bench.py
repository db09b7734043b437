"""Decode time per image of the VAE decoder, fp16 against bf16 engines, from random-init weights.

Shapes: the SD VAE at 512^2 (64^2 latents) and the SDXL VAE at 768^2 and 1024^2.  Both engines of one shape are built
in the same process and timed alternately (CUDA events around `--iters` eager decodes after `--warmup` decodes, `--rounds`
rounds), so clock or thermal drift hits both alike.  Prints the card name and power limit with the numbers.

    python tools/vae_bench.py [--iters 10] [--warmup 3] [--rounds 3]
"""
import argparse
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import torch  # noqa: E402


def _power_limit():
    try:
        r = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader"], capture_output=True,
                           text=True, timeout=20)
        return r.stdout.strip().splitlines()[0]
    except Exception:  # noqa: BLE001 -- informational only
        return "unknown"


def _time(eng, z, iters, warmup):
    for _ in range(warmup):
        eng.forward(z)
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(iters):
        eng.forward(z)
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / iters


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--rounds", type=int, default=3)
    args = ap.parse_args()
    from b200sd import config as C
    from b200sd import lib
    from b200sd.vae import VAEDecoderEngine

    lib.load()
    print(f"# {torch.cuda.get_device_name(0)}, power limit {_power_limit()}")
    for name, cfg, lat in (("SD VAE", C.SD_VAE, 64), ("SDXL VAE", C.SDXL_VAE, 96), ("SDXL VAE", C.SDXL_VAE, 128)):
        sd = C.random_state_dict(C.vae_decoder_param_shapes(cfg), seed=1, dtype=torch.float16)
        engines = {dt: VAEDecoderEngine(cfg, sd, "cuda", dtype=dt) for dt in (torch.float16, torch.bfloat16)}
        z = torch.randn(1, 4, lat, lat, generator=torch.Generator().manual_seed(2)).cuda()
        times = {dt: [] for dt in engines}
        for _ in range(args.rounds):
            for dt, eng in engines.items():
                times[dt].append(_time(eng, z, args.iters, args.warmup))
        f16, bf16 = (", ".join(f"{t:.2f}" for t in times[dt]) for dt in engines)
        print(f"{name} {8 * lat}^2: fp16 {f16} ms/image; bf16 {bf16} ms/image "
              f"(median ratio bf16/fp16 {sorted(times[torch.bfloat16])[len(times[torch.bfloat16]) // 2] / sorted(times[torch.float16])[len(times[torch.float16]) // 2]:.3f})")
        del engines
        torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
