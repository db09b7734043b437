"""fp16 against W8A8 UNet on the device loop: loop-graph iterations per second, alternating the two precisions; per
launch class (GEMM / convolution, attention, normalisation, elementwise) ms per step from loop graphs captured with
only that class launching (bench.py's mechanism); per quantized layer the 3x3 convolution launch in fp16 and in int8
from CUDA events over a graph of repeated launches; and the PSNR of the W8A8 final latents against fp16.  Random-init
weights (no checkpoint exists offline): the PSNR says nothing about the image quality of a trained checkpoint.
--linear: the recipe also quantizes every transformer linear; the loop runs fp16, convolutions-only and convolutions +
linears alternated, and the per-layer table covers the int8 linear launches (with the LayerNorm -> int8 launch that
feeds attn1.to_q|k|v, attn2.to_q and ff.net.0.proj) against the fp16 linear of the same shape.

    python tools/w8a8_bench.py --model sd21-base --size 512 --steps 20 --rounds 3 [--linear] --out DIR
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


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--model", default="sd21-base", choices=["sd21-base", "sdxl-base"])
    ap.add_argument("--size", type=int, default=512)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--calib-steps", type=int, default=10)
    ap.add_argument("--linear", action="store_true")
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("w8a8_bench needs a GPU")
    from b200sd import config as C
    from b200sd import lib as L
    from b200sd.model import UNetModel
    from b200sd.pipeline import B200StableDiffusionPipeline as P
    from b200sd.quantization import compute_psnr

    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm,clocks.sm", "--format=csv,noheader"],
                         capture_output=True, text=True).stdout.strip()
    pipe = P.from_random_init(args.model, images_per_call=1, seed=0, height=args.size, width=args.size)
    cfg = {"sd21-base": C.SD21_BASE_UNET, "sdxl-base": C.SDXL_BASE_UNET}[args.model]
    recipe = pipe.calibrate_unet(["a photograph of an astronaut riding a horse"], num_inference_steps=args.calib_steps,
                                 seed=1, linear=args.linear)
    u16 = pipe.unet
    usd = C.random_state_dict(C.unet_param_shapes(cfg), seed=0, dtype=torch.float16)  # from_random_init's UNet weights
    u8 = UNetModel(cfg, usd, batch=u16.batch, height=u16.h, width=u16.w, quantization=recipe)
    models = {"fp16": u16, "w8a8": u8}
    if args.linear:
        models = {"fp16": u16, "w8a8_convs": UNetModel(cfg, usd, batch=u16.batch, height=u16.h, width=u16.w,
                                                       quantization=recipe.subset(recipe.scales)),
                  "w8a8_convs_linears": u8}
    del usd
    xl = u16.engine.xl
    g = np.random.RandomState(0)
    lat = torch.from_numpy(g.randn(1, 4, u16.h, u16.w).astype(np.float32))
    emb = torch.from_numpy((g.randn(2, cfg["cross_attention_dim"], 1, 77) * 0.5).astype(np.float16))
    kw = {}
    if xl:
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

    res = {name: [] for name in models}
    outs = {}
    for _ in range(args.rounds):
        for name, unet in models.items():
            ips, outs[name] = run(unet)
            res[name].append(ips)

    lib = L.load()
    classes = {"gemm_conv": 1, "attention": 2, "normalisation": 4, "elementwise": 8}
    per_class = {name: {} for name in models}
    for name, unet in models.items():
        run(unet)  # the full graph first: workspaces, weight tiling and kernel attributes exist before a class capture
        for cname, bit in classes.items():
            pipe._loop_graphs = {}
            lib.b200sd_set_launch_classes(bit)
            try:
                pipe.denoise(emb, lat, args.steps, 7.5, **kw)  # captures the class-only loop graph
            finally:
                lib.b200sd_set_launch_classes(0xF)
            torch.cuda.synchronize()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            for _ in range(3):
                pipe.denoise(emb, lat, args.steps, 7.5, **kw)  # replays it
            e1.record()
            torch.cuda.synchronize()
            per_class[name][cname] = e0.elapsed_time(e1) / (3 * args.steps)
    pipe._loop_graphs = {}

    # per layer: record the int8 launches of one forward, then time each launch and its fp16 twin
    calls, lcalls, ln_out = [], [], {}
    orig, orig_lin, orig_ln = L.conv3x3_s8, L.linear_s8, L.layer_norm_s8

    def record(x, wgt, col_scale, bias=None, residual=None, **k):
        calls.append((x, wgt, col_scale, bias, residual, k))
        return orig(x, wgt, col_scale, bias, residual, **k)

    def record_lin(x, wgt, col_scale, bias=None, residual=None, **k):
        lcalls.append((x, wgt, col_scale, bias, residual, k, ln_out.get(x.data_ptr())))
        return orig_lin(x, wgt, col_scale, bias, residual, **k)

    def record_ln(x, gamma, beta, inv_scale, eps=1e-5, out=None):
        q = orig_ln(x, gamma, beta, inv_scale, eps, out)
        ln_out[q.data_ptr()] = (x, gamma, beta, inv_scale)
        return q

    L.conv3x3_s8, L.linear_s8, L.layer_norm_s8 = record, record_lin, record_ln
    graphed, u8.use_cuda_graph = u8.use_cuda_graph, False
    try:
        pipe.unet = u8
        pipe.denoise(emb, lat, 1, 7.5, record=[], **kw)  # one eager UNet call
    finally:
        L.conv3x3_s8, L.linear_s8, L.layer_norm_s8 = orig, orig_lin, orig_ln
        u8.use_cuda_graph = graphed
    names = [n for n in recipe.scales]
    calls = calls[:len(names)]

    def time_us(fn, reps=20):
        fn()
        torch.cuda.synchronize()
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g):
            for _ in range(reps):
                fn()
        g.replay()
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(5):
            g.replay()
        e1.record()
        torch.cuda.synchronize()
        return 1000.0 * e0.elapsed_time(e1) / (5 * reps)

    layers = []
    gen = torch.Generator(device="cuda").manual_seed(0)
    for layer, (x8, w8, cs, bias, residual, k) in zip(names, calls):
        n, h, w, c = x8.shape
        x16 = torch.randn(n, h, w, c, device="cuda", generator=gen).half()
        w16 = (torch.randn(w8.shape[0], w8.shape[1], device="cuda", generator=gen) * 0.02).half()
        t8 = time_us(lambda: orig(x8, w8, cs, bias, residual, **k))
        t16 = time_us(lambda: L.conv3x3(x16, w16, bias, residual, bias_rows=k.get("bias_rows", 0),
                                        bias_stride=k.get("bias_stride", 0)))
        layers.append({"layer": layer, "hw": h, "cin": c, "cout": w8.shape[0], "fp16_us": round(t16, 2),
                       "int8_us": round(t8, 2), "int8_over_fp16": round(t8 / t16, 3)})
        print(json.dumps(layers[-1]), flush=True)
    # linear launches: the int8 GEMM (+ the LayerNorm -> int8 launch that feeds it) against the fp16 GEMM of that shape
    # (the fp16 model folds that LayerNorm into the GEMM: no launch of its own)
    linears = []
    for x8, w8, cs, bias, residual, k, ln in lcalls:
        m, c = x8.shape
        geglu = k.get("geglu", False)
        x16 = torch.randn(m, c, device="cuda", generator=gen).half()
        w16 = (torch.randn(w8.shape[0], c, device="cuda", generator=gen) * 0.02).half()
        t8 = time_us(lambda: orig_lin(x8, w8, cs, bias, residual, **k))
        tln = time_us(lambda: orig_ln(*ln)) if ln is not None else 0.0
        t16 = time_us(lambda: L.linear(x16, w16, bias, residual, geglu=geglu, static_w=True))
        linears.append({"m": m, "k": c, "n": w8.shape[0], "geglu": geglu, "int8_out": k.get("out_inv_scale") is not None,
                        "fp16_us": round(t16, 2), "int8_us": round(t8, 2), "layer_norm_s8_us": round(tln, 2),
                        "int8_total_over_fp16": round((t8 + tln) / t16, 3)})
    by_shape = {}
    for d in linears:
        by_shape.setdefault((d["m"], d["k"], d["n"], d["geglu"], d["int8_out"], d["layer_norm_s8_us"] > 0), []).append(d)
    linear_table = [dict(v[0], launches=len(v)) for v in by_shape.values()]
    for d in linear_table:
        print(json.dumps(d), flush=True)
    line = {"gpu": gpu, "model": args.model, "size": args.size, "unet_batch": 2, "steps": args.steps,
            "iter_per_s": res, "class_ms_per_step": per_class, "quantized_layers": len(recipe),
            "layers_int8_slower": [d["layer"] for d in layers if d["int8_us"] > d["fp16_us"]],
            "layers": layers, "linear_launches": linear_table,
            "linear_launches_int8_slower": sum(d["launches"] for d in linear_table if d["int8_total_over_fp16"] > 1),
            "psnr_w8a8_vs_fp16_latents_random_init": {n: compute_psnr(outs["fp16"].cpu(), o.cpu())
                                                      for n, o in outs.items() if n != "fp16"}}
    print(json.dumps(line))
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        tag = "_linear" if args.linear else ""
        with open(os.path.join(args.out, f"w8a8_bench_{args.model}_{args.size}{tag}.json"), "w") as f:
            json.dump(line, f, indent=1)


if __name__ == "__main__":
    main()
