"""fp16 against palettized UNet weights.  Per distinct palettized launch shape of one UNet forward (the launches of a
uniform 4-bit engine): the fp16 kernel on fp16 weights against b200sd_gemm_lut at 8, 6 and 4 bits, from CUDA events
over a graph of repeated launches; whole-loop iterations per second of the device loop for fp16, uniform 4-bit and a
mixed recipe in alternating rounds; each engine's weight_bytes and the device memory its build and first loop added;
and the PSNR of the palettized final latents against fp16.  Random-init weights (no checkpoint exists offline): the
PSNR says nothing about the image quality of a trained checkpoint.

    python tools/palettization_bench.py --model sd21-base --size 512 --steps 20 --rounds 3 --out DIR
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))


def mixed_recipe(cfg):
    """A fixed mixed recipe (not one of Apple's, which need a trained checkpoint's PSNR analysis): attention
    projections at 6 bits, feed-forward and convolutions at 4, proj_in / proj_out and the embeddings at 8."""
    from b200sd import palettization as Pz

    out = {}
    for name in Pz.palettizable_layers(cfg):
        if ".attn" in name:
            out[name] = 6
        elif "proj_in" in name or "proj_out" in name or "embedding" in name or "time_emb_proj" in name:
            out[name] = 8
        else:
            out[name] = 4
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--model", default="sd21-base", choices=["sd21-base", "sdxl-base"])
    ap.add_argument("--size", type=int, default=512)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("palettization_bench needs a GPU")
    from b200sd import config as C
    from b200sd import lib as L
    from b200sd import palettization as Pz
    from b200sd.model import UNetModel
    from b200sd.pipeline import B200StableDiffusionPipeline as P
    from b200sd.quantization import compute_psnr

    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm,clocks.sm", "--format=csv,noheader"],
                         capture_output=True, text=True).stdout.strip()
    cfg = {"sd21-base": C.SD21_BASE_UNET, "sdxl-base": C.SDXL_BASE_UNET}[args.model]
    mem = {}
    pipe = P.from_random_init(args.model, images_per_call=1, seed=0, height=args.size, width=args.size)
    u16 = pipe.unet
    usd = C.random_state_dict(C.unet_param_shapes(cfg), seed=0, dtype=torch.float16)  # from_random_init's UNet weights
    g = np.random.RandomState(0)
    lat = torch.from_numpy(g.randn(1, 4, u16.h, u16.w).astype(np.float32))
    emb = torch.from_numpy((g.randn(2, cfg["cross_attention_dim"], 1, 77) * 0.5).astype(np.float16))
    kw = {}
    if u16.engine.xl:
        kw = dict(time_ids=torch.tensor([[args.size, args.size, 0, 0, args.size, args.size]] * 2, dtype=torch.float16,
                                        device="cuda"),
                  text_embeds=torch.from_numpy((g.randn(2, C.SDXL_POOLED_DIM) * 0.5).astype(np.float16)).cuda())

    def run(unet):
        pipe.unet = unet
        pipe._loop_graphs = {}
        out = pipe.denoise(emb, lat, args.steps, 7.5, **kw).clone()  # captures the loop graph
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        out = pipe.denoise(emb, lat, args.steps, 7.5, **kw).clone()
        torch.cuda.synchronize()
        return args.steps / (time.perf_counter() - t0), out

    def resident(build):
        torch.cuda.synchronize()
        a = torch.cuda.memory_allocated()
        unet = build()
        run(unet)
        torch.cuda.synchronize()
        return unet, torch.cuda.memory_allocated() - a

    recipes = {"uniform4": 4, "mixed": mixed_recipe(cfg)}
    unets = {}
    for name, rec in [("fp16", None)] + list(recipes.items()):
        unets[name], mem[name] = resident(lambda: UNetModel(cfg, usd, batch=u16.batch, height=u16.h, width=u16.w,
                                                          palettization=rec))
    del usd
    res = {k: [] for k in unets}
    outs = {}
    for _ in range(args.rounds):
        for name, unet in unets.items():
            ips, outs[name] = run(unet)
            res[name].append(round(ips, 2))
    pipe._loop_graphs = {}

    # the palettized launches of one eager forward of the 4-bit engine, one entry per distinct shape
    calls = {}
    orig = {"linear": L.linear, "conv3x3": L.conv3x3}

    def recorder(kind):
        def rec(x, wgt, *a, **k):
            if isinstance(wgt, Pz.PalettizedWeight):
                key = (kind, tuple(x.shape), wgt.shape, wgt.kscale is not None, bool(k.get("geglu")),
                       len(a) > 1 and a[1] is not None, k.get("x1") is not None, k.get("stride", 1))
                if key not in calls:
                    calls[key] = [x, wgt, a, dict(k), 0]
                calls[key][4] += 1
            return orig[kind](x, wgt, *a, **k)
        return rec

    u4 = unets["uniform4"]
    L.linear, L.conv3x3 = recorder("linear"), recorder("conv3x3")
    graphed, u4.use_cuda_graph = u4.use_cuda_graph, False
    try:
        pipe.unet = u4
        pipe.denoise(emb, lat, 1, 7.5, record=[], **kw)
    finally:
        L.linear, L.conv3x3 = orig["linear"], orig["conv3x3"]
        u4.use_cuda_graph = graphed
    pipe._loop_graphs = {}

    def time_us(fn, reps=20):
        fn()
        torch.cuda.synchronize()
        gr = torch.cuda.CUDAGraph()
        with torch.cuda.graph(gr):
            for _ in range(reps):
                fn()
        gr.replay()
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(5):
            gr.replay()
        e1.record()
        torch.cuda.synchronize()
        return 1000.0 * e0.elapsed_time(e1) / (5 * reps)

    layers = []
    for (kind, xs, ws, folded, geglu, res_, two, stride), (x, pw, a, k, count) in calls.items():
        fn = orig[kind]
        w16 = pw.decoded()
        if kind == "linear":
            k16 = dict(k, static_w=True)
        else:
            k16 = dict(k)
        row = {"kind": kind, "x": list(xs), "w": list(ws), "launches_per_forward": count, "ln_fold": folded,
               "geglu": geglu, "residual": res_, "fp16_us": round(time_us(lambda: fn(x, w16, *a, **k16)), 2)}
        # a folded launch's palette is fit on the unscaled weight, as the engine does
        base = w16 if pw.kscale is None else (w16.float() / pw.kscale[None, :]).half()
        for nb in (8, 6, 4):
            fit = Pz.fit_palette(base, nb)
            pwn = Pz.palettized([(fit[0], fit[1], nb)], pw.kscale)
            row[f"lut{nb}_us"] = round(time_us(lambda: fn(x, pwn, *a, **k)), 2)
        row["lut4_over_fp16"] = round(row["lut4_us"] / row["fp16_us"], 3)
        layers.append(row)
        print(json.dumps(row), flush=True)
    line = {"gpu": gpu, "model": args.model, "size": args.size, "unet_batch": 2, "steps": args.steps,
            "iter_per_s": res, "weight_bytes": {k: u.engine.weight_bytes for k, u in unets.items()},
            "resident_bytes": mem, "nominal_bits": {"uniform4": 4.0, "mixed": Pz.nominal_bits(recipes["mixed"], cfg)},
            "psnr_vs_fp16_latents_random_init": {k: compute_psnr(outs["fp16"].cpu(), outs[k].cpu()) for k in recipes},
            "fp16_kernel_us_per_forward": round(sum(r["fp16_us"] * r["launches_per_forward"] for r in layers), 1),
            "lut_kernel_us_per_forward": {nb: round(sum(r[f"lut{nb}_us"] * r["launches_per_forward"] for r in layers), 1)
                                          for nb in (8, 6, 4)},
            "layers": layers}
    print(json.dumps({k: v for k, v in line.items() if k != "layers"}))
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, f"palettization_bench_{args.model}_{args.size}.json"), "w") as f:
            json.dump(line, f, indent=1)


if __name__ == "__main__":
    main()
