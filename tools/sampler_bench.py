"""Per-step time of the whole-loop CUDA graph for each scheduler, and of the noised step kernel alone.

    python tools/sampler_bench.py [--reps 5] [--steps 20]

Workload: random-init SD-2.1-base, txt2img 512x512 at UNet batch 2 (uncond, cond), 20 steps, CFG 7.5.  For each of the
six schedulers the 20-step loop (with its per-prompt prologue) is captured once by ``pipe.denoise`` and replayed
``--reps`` times between CUDA events; ms per step = elapsed / (reps * steps).  Each scheduler is measured twice, in
two rounds, so the run-to-run spread is visible next to the differences.  The step kernel alone:
``b200sd_cfg_scheduler_step_noised`` (and the plain step for comparison) captured 100 times into one CUDA graph at
1x4x64x64 and 8x4x64x64 latents, µs per launch.  Prints one JSON line with the card name and power limit."""
import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import numpy as np  # noqa: E402
import torch  # noqa: E402

SCHEDULERS = ("DDIM", "DPMSolverMultistep", "PNDM", "EulerDiscrete", "EulerAncestralDiscrete", "LMSDiscrete")


def power_limit_w(index):
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader,nounits", "-i", str(index)],
                             stdout=subprocess.PIPE, stderr=subprocess.DEVNULL, text=True, timeout=10).stdout.strip()
        return float(out)
    except Exception:
        return None


def loop_ms_per_step(pipe, emb, lat, steps, reps):
    pipe.denoise(emb, lat, steps, 7.5, noise_key=1)  # capture + warm-up
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for r in range(reps):
        pipe.denoise(emb, lat, steps, 7.5, noise_key=r)
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / (reps * steps)


def step_kernel_us(L, n, noised, launches=100):
    from b200sd import scheduler as S
    from b200sd.pipeline import B200StableDiffusionPipeline as P
    eps = torch.randn(2 * n, 4, 64, 64, device="cuda")
    lat = torch.randn(n, 4, 64, 64, device="cuda")
    hist = torch.zeros(4, n, 4, 64, 64, device="cuda")
    unet_in = torch.zeros(2 * n, 64, 64, 8, dtype=torch.float16, device="cuda")
    key = torch.tensor([7], dtype=torch.int32, device="cuda")
    st = S.EulerAncestralDiscreteScheduler(20).plan()[3]
    k = P._coeffs(st, 7.5)

    def run():
        for i in range(launches):
            if noised:
                L.cfg_scheduler_step_noised(eps, lat, k, st.noise_scale, key, i, hist=hist, unet_in=unet_in)
            else:
                L.cfg_scheduler_step(eps, lat, k, hist=hist, unet_in=unet_in)

    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        run()
    torch.cuda.current_stream().wait_stream(s)
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        run()
    g.replay()
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    reps = 20
    a.record()
    for _ in range(reps):
        g.replay()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) * 1e3 / (reps * launches)


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n")[0])
    ap.add_argument("--reps", type=int, default=5, help="replays of the 20-step loop per measurement")
    ap.add_argument("--steps", type=int, default=20)
    args = ap.parse_args()

    from b200sd import lib as L
    from b200sd.pipeline import B200StableDiffusionPipeline

    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    L.load()
    pipe = B200StableDiffusionPipeline.from_random_init("sd21-base", images_per_call=1, device=dev, seed=1)
    d_ctx = pipe.unet._ctx.shape[1]
    g = torch.Generator().manual_seed(93)
    emb = torch.cat([torch.zeros(1, d_ctx, 1, 77), torch.randn(1, d_ctx, 1, 77, generator=g)]).half().to(dev)
    lat = torch.randn(1, 4, 64, 64, generator=g).half().float().to(dev)
    rounds = {name: [] for name in SCHEDULERS}
    for _ in range(2):
        for name in SCHEDULERS:
            pipe.scheduler_name = name
            pipe.scheduler_kwargs = {"final_sigmas_type": "zero"} if name == "DPMSolverMultistep" else {}
            rounds[name].append(round(loop_ms_per_step(pipe, emb, lat * pipe_init_sigma(name, args.steps),
                                                       args.steps, args.reps), 4))
    kernel = {f"{n}x4x64x64": {"noised_us": round(step_kernel_us(L, n, True), 3),
                               "plain_us": round(step_kernel_us(L, n, False), 3)} for n in (1, 8)}
    print(json.dumps({"workload": f"SD-2.1-base txt2img 512x512, UNet batch 2, {args.steps} steps, CFG 7.5, fp16",
                      "loop_ms_per_step": rounds, "step_kernel_100_graph_launches": kernel,
                      "card": torch.cuda.get_device_name(dev), "power_limit_w": power_limit_w(0)}), flush=True)


def pipe_init_sigma(name, steps):
    from b200sd import scheduler as S
    return float(np.float32(S.make_scheduler(name, steps).init_noise_sigma))


if __name__ == "__main__":
    main()
