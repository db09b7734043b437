"""Iter/s of the device denoising loop for one model, with the attention kernels' share of a step.

    python tools/model_bench.py --model sd15|sd21-base|sd21 [--reps 3]
    python tools/model_bench.py --inpaint [--rounds 5] [--reps 3]
    python tools/model_bench.py --guidance-free --model sd21-base|sdxl-base [--rounds 5] [--reps 3]
    python tools/model_bench.py --controlnet [--rounds 5] [--reps 3]

The workload is bench.py's: random-init weights, txt2img 512x512 at UNet batch 2 (uncond, cond), 20 DDIM steps, CFG
7.5, the 20 steps (with the per-prompt prologue) captured as one CUDA graph by bench.LoopBench and timed with
bench.timed_replays.  ``sd21`` (SD 2.0 / 2.1 768-v) runs the same UNet at 768x768 (96x96 latents) with 20 DDIM
v-prediction steps.  The attention time is the same loop captured with only the attention class launching
(classes=2).  Prints one JSON line: iter/s, ms per step, attention ms per step, card name, power limit and the median
SM clock while the loop ran.

``--guidance-free`` (512x512, random-init weights): the pipeline's 20-step DDIM loop graph with CFG 7.5 (UNet batch 2)
against the same loop guidance-free (guidance 1.0, UNet batch 1), and the whole ``__call__`` (text encoding, the loop,
VAE decode; output_type "np") of a 1-step Euler-ancestral (trailing) call at guidance 0 and a 4-step LCM call (the
UNet with time_cond_proj_dim=256), alternated ``--rounds`` times.  One JSON line per mode.

``--controlnet``: SDXL-base at 1024x1024 (random-init weights), the pipeline's 20-step DDIM loop graph at CFG 5 (UNet
batch 2) with 0, 1 and 2 random-init SDXL ControlNets (config.SDXL_CONTROLNET, scale 0.5) running at every step,
alternated ``--rounds`` times, and one SDXL ControlNet forward at batch 2 alone (its own CUDA graph, CUDA events).
One JSON line: ms per step of each loop, the ControlNet forward, and the 1-net loop less the 0-net loop."""
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


def inpaint_modes(args, dev):
    """SD-1.5 512x512, UNet batch 2, 20 DDIM steps, CFG 7.5: the pipeline's own loop graph for text-to-image, for
    inpainting with the 4-channel blend, and for a 9-channel inpainting UNet, timed alternately ``--rounds`` times."""
    import numpy as np

    from b200sd import config as C
    from b200sd.pipeline import B200StableDiffusionPipeline as P
    from b200sd.pipeline import InpaintInputs

    n = bench.N_STEPS_IMG
    p4 = P.from_random_init("sd15", images_per_call=1, device=dev, seed=1, scheduler="DDIM")
    p9 = P.from_random_init("sd15", images_per_call=1, device=dev, seed=1, scheduler="DDIM",
                            unet_cfg=dict(C.SD15_UNET, in_channels=9))
    g = torch.Generator().manual_seed(93)
    emb = torch.cat([torch.zeros(1, 768, 1, 77), torch.randn(1, 768, 1, 77, generator=g)]).half()
    lat = torch.randn(1, 4, 64, 64, generator=g).half().float()
    mask = (torch.rand(1, 1, 64, 64, generator=g) > 0.5).float()
    inp = InpaintInputs(mask, torch.randn(1, 4, 64, 64, generator=g), lat, torch.randn(1, 4, 64, 64, generator=g))
    graphs = {}
    for mode, pipe, extra in (("txt2img", p4, None), ("inpaint-blend", p4, inp), ("inpaint-9ch", p9, inp)):
        before = set(pipe._loop_graphs)
        pipe.denoise(emb, lat, n, 7.5, inpaint=extra)
        key, = set(pipe._loop_graphs) - before
        graphs[mode] = pipe._loop_graphs[key]
    sync = torch.cuda.synchronize
    times = {m: [] for m in graphs}
    sampler = bench.ClockSampler(0)
    sampler.start()
    for _ in range(args.rounds):
        for mode, graph in graphs.items():
            times[mode].append(bench.timed_replays(graph, args.reps, sync) / n)
    clocks = sampler.stop()
    for mode, ms in times.items():
        med = float(np.median(ms))
        print(json.dumps({"model": "sd15", "mode": mode,
                          "workload": "512x512, UNet batch 2, 20 DDIM steps, CFG 7.5, fp16, pipeline loop graph",
                          "iter_per_s": round(1e3 / med, 2), "ms_per_step": round(med, 4),
                          "ms_per_step_rounds": [round(v, 4) for v in ms],
                          "card": torch.cuda.get_device_name(dev), "power_limit_w": power_limit_w(0),
                          "sm_mhz": clocks.get("sm_mhz"), "clock_events": clocks.get("reasons")}), flush=True)


def guidance_free_modes(args, dev):
    import time

    import numpy as np

    from b200sd import config as C
    from b200sd.pipeline import B200StableDiffusionPipeline as P

    model = args.model
    base = {"sd21-base": C.SD21_BASE_UNET, "sdxl-base": C.SDXL_BASE_UNET}[model]
    ddim = P.from_random_init(model, device=dev, seed=1, scheduler="DDIM")
    turbo = P.from_random_init(model, device=dev, seed=1, scheduler="EulerAncestralDiscrete",
                               scheduler_kwargs={"timestep_spacing": "trailing"})
    lcm = P.from_random_init(model, device=dev, seed=1, scheduler="LCM",
                             unet_cfg=dict(base, time_cond_proj_dim=256))
    g = torch.Generator().manual_seed(93)
    d_ctx = ddim.unet._ctx.shape[1]
    emb = torch.cat([torch.zeros(1, d_ctx, 1, 77), torch.randn(1, d_ctx, 1, 77, generator=g)]).half()
    lat = torch.randn(1, 4, 64, 64, generator=g).half().float()
    kw = {}
    if ddim.xl:
        kw = dict(time_ids=torch.tensor([[512.0, 512.0, 0.0, 0.0, 512.0, 512.0]] * 2),
                  text_embeds=torch.randn(2, 1280, generator=g))
    n = bench.N_STEPS_IMG
    graphs = {}
    for mode, gs in (("ddim20-cfg-b2", 7.5), ("ddim20-guidance-free-b1", 1.0)):
        before = set(ddim._loop_graphs)
        ddim.denoise(emb, lat, n, gs, **kw)
        key, = set(ddim._loop_graphs) - before
        graphs[mode] = ddim._loop_graphs[key]
    calls = {"euler-a-trailing-1step-call": lambda: turbo("a cat", num_inference_steps=1, guidance_scale=0.0, seed=1,
                                                         output_type="np"),
             "lcm-4step-call": lambda: lcm("a cat", num_inference_steps=4, guidance_scale=8.0, seed=1,
                                           output_type="np")}
    for fn in calls.values():  # warm-up: loop graphs, workspaces
        fn()
        fn()
    sync = torch.cuda.synchronize
    times = {m: [] for m in list(graphs) + list(calls)}
    sampler = bench.ClockSampler(0)
    sampler.start()
    for _ in range(args.rounds):
        for mode, graph in graphs.items():
            times[mode].append(bench.timed_replays(graph, args.reps, sync) / n)
        for mode, fn in calls.items():
            ms = []
            for _ in range(args.reps):
                sync()
                t0 = time.perf_counter()
                fn()
                sync()
                ms.append((time.perf_counter() - t0) * 1e3)
            times[mode].append(float(np.median(ms)))
    clocks = sampler.stop()
    for mode, ms in times.items():
        med = float(np.median(ms))
        rec = {"model": model, "mode": mode, "workload": "512x512, random-init weights, fp16"}
        if mode in graphs:
            rec.update(iter_per_s=round(1e3 / med, 2), ms_per_step=round(med, 4),
                       ms_per_step_rounds=[round(v, 4) for v in ms])
        else:
            rec.update(ms_per_call=round(med, 3), ms_per_call_rounds=[round(v, 3) for v in ms])
        rec.update(card=torch.cuda.get_device_name(dev), power_limit_w=power_limit_w(0), sm_mhz=clocks.get("sm_mhz"),
                   clock_events=clocks.get("reasons"))
        print(json.dumps(rec), flush=True)


def controlnet_modes(args, dev):
    import numpy as np

    from b200sd import config as C
    from b200sd.pipeline import B200StableDiffusionPipeline as P

    two = P.from_random_init("sdxl-base", device=dev, seed=1, scheduler="DDIM", height=1024, width=1024,
                             controlnet_cfgs=[C.SDXL_CONTROLNET] * 2)
    one = P(two.unet, two.vae_decoder, scheduler="DDIM", xl=True, controlnet=two.controlnet[:1])
    g = torch.Generator().manual_seed(93)
    emb = torch.cat([torch.zeros(1, 2048, 1, 77), torch.randn(1, 2048, 1, 77, generator=g)]).half()
    lat = torch.randn(1, 4, 128, 128, generator=g).half().float()
    kw = dict(time_ids=torch.tensor([[1024.0, 1024.0, 0.0, 0.0, 1024.0, 1024.0]] * 2),
              text_embeds=torch.randn(2, 1280, generator=g))
    cond = [torch.rand(2, 3, 1024, 1024, generator=g).half() for _ in range(2)]
    n = bench.N_STEPS_IMG
    graphs = {}
    for mode, pipe, cc in (("0-controlnets", two, None), ("1-controlnet", one, cond[:1]), ("2-controlnets", two, cond)):
        before = set(pipe._loop_graphs)
        pipe.denoise(emb, lat, n, 5.0, controlnet_cond=cc, controlnet_conditioning_scale=0.5, **kw)
        key, = set(pipe._loop_graphs) - before
        graphs[mode] = pipe._loop_graphs[key]
    # one ControlNet forward alone: the model's own graph on the static inputs the last loop left behind
    cn = two.controlnet[0]
    cn.forward_device()
    sync = torch.cuda.synchronize
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    times = {m: [] for m in list(graphs) + ["controlnet-forward"]}
    sampler = bench.ClockSampler(0)
    sampler.start()
    for _ in range(args.rounds):
        for mode, graph in graphs.items():
            times[mode].append(bench.timed_replays(graph, args.reps, sync) / n)
        sync()
        e0.record()
        for _ in range(n * args.reps):
            cn.forward_device()
        e1.record()
        sync()
        times["controlnet-forward"].append(e0.elapsed_time(e1) / (n * args.reps))
    clocks = sampler.stop()
    med = {m: float(np.median(v)) for m, v in times.items()}
    print(json.dumps({"model": "sdxl-base + SDXL ControlNet",
                      "workload": "1024x1024, random-init weights, UNet / ControlNet batch 2, 20 DDIM steps, CFG 5, "
                                  "conditioning scale 0.5, fp16, pipeline loop graph",
                      "ms_per_step": {m: round(v, 4) for m, v in med.items()},
                      "ms_per_step_rounds": {m: [round(x, 4) for x in v] for m, v in times.items()},
                      "controlnet_cost_in_loop_ms": round(med["1-controlnet"] - med["0-controlnets"], 4),
                      "second_controlnet_cost_in_loop_ms": round(med["2-controlnets"] - med["1-controlnet"], 4),
                      "card": torch.cuda.get_device_name(dev), "power_limit_w": power_limit_w(0),
                      "sm_mhz": clocks.get("sm_mhz"), "clock_events": clocks.get("reasons")}), flush=True)


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n")[0])
    ap.add_argument("--model", choices=("sd15", "sd21-base", "sd21", "sdxl-base"), default="sd15",
                    help="sdxl-base: --guidance-free only")
    ap.add_argument("--reps", type=int, default=3, help="replays of the 20-step graph per measurement")
    ap.add_argument("--inpaint", action="store_true", help="SD-1.5: text-to-image vs the two inpainting loops")
    ap.add_argument("--rounds", type=int, default=5, help="--inpaint / --guidance-free: alternated measurements per mode")
    ap.add_argument("--guidance-free", action="store_true",
                    help="--model sd21-base | sdxl-base: the CFG loop against the guidance-free one, Turbo / LCM calls")
    ap.add_argument("--controlnet", action="store_true",
                    help="SDXL-base 1024x1024: the loop with 0, 1 and 2 SDXL ControlNets, one ControlNet forward alone")
    args = ap.parse_args()
    if args.controlnet:
        dev = torch.device("cuda", 0)
        torch.cuda.set_device(dev)
        controlnet_modes(args, dev)
        return
    if args.guidance_free:
        if args.model not in ("sd21-base", "sdxl-base"):
            ap.error("--guidance-free runs --model sd21-base or sdxl-base")
        dev = torch.device("cuda", 0)
        torch.cuda.set_device(dev)
        guidance_free_modes(args, dev)
        return
    if args.model == "sdxl-base":
        ap.error("--model sdxl-base runs with --guidance-free only")
    if args.inpaint:
        dev = torch.device("cuda", 0)
        torch.cuda.set_device(dev)
        inpaint_modes(args, dev)
        return

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
