"""Tuning aid for plan_gemm's cost model: times the GEMM / conv shapes of the SD-2.1 UNet at a 512x512 image, batch 2
(every resolution level, the qkv and GEGLU projections included) for every (block_n, split, cluster|workspace)
candidate, weights rotated through > L2 bytes."""
import json
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch  # noqa: E402

from b200sd import lib as L  # noqa: E402

SHAPES = [  # (name, mode, n_img, h, c0, c1, cout)   mode 1 = conv3x3 at h x h, mode 0 = linear with M = n_img*h*h
    ("conv64_320", 1, 2, 64, 320, 0, 320), ("conv64_640", 1, 2, 64, 320, 320, 320), ("conv64_960", 1, 2, 64, 640, 320, 320),
    ("lin8192_320", 0, 2, 64, 320, 0, 320), ("lin8192_1280", 0, 2, 64, 1280, 0, 320),
    ("qkv8192_960", 0, 2, 64, 320, 0, 960), ("geglu8192_2560", 0, 2, 64, 320, 0, 2560),
    ("qkv2048_1920", 0, 2, 32, 640, 0, 1920), ("geglu2048_5120", 0, 2, 32, 640, 0, 5120),
    ("qkv512_3840", 0, 2, 16, 1280, 0, 3840), ("geglu512_10240", 0, 2, 16, 1280, 0, 10240),
    ("conv8_1280", 1, 2, 8, 1280, 0, 1280), ("conv8_2560", 1, 2, 8, 1280, 1280, 1280),
    ("conv16_1280", 1, 2, 16, 1280, 0, 1280), ("conv16_1920", 1, 2, 16, 1280, 640, 1280),
    ("conv16_2560", 1, 2, 16, 1280, 1280, 1280), ("conv16_640_1280", 1, 2, 16, 640, 0, 1280),
    ("conv32_640", 1, 2, 32, 640, 0, 640), ("conv32_1280", 1, 2, 32, 640, 640, 640), ("conv32_960", 1, 2, 32, 640, 320, 640),
    ("conv32_1920", 1, 2, 32, 1280, 640, 640), ("conv32_320_640", 1, 2, 32, 320, 0, 640),
    ("lin512_1280", 0, 2, 16, 1280, 0, 1280), ("lin512_5120", 0, 2, 16, 5120, 0, 1280),
    ("lin128_1280", 0, 2, 8, 1280, 0, 1280), ("lin128_5120", 0, 2, 8, 5120, 0, 1280),
    ("lin2048_640", 0, 2, 32, 640, 0, 640), ("lin2048_2560", 0, 2, 32, 2560, 0, 640),
]
BNS = [32, 64, 96, 128, 160, 192, 256]  # the compiled tile widths (16: N < 32 only)


def time_graph(fn, ncopies, reps=6):
    for i in range(ncopies):
        fn(i)
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        for i in range(ncopies):
            fn(i)
    g.replay()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(reps):
        g.replay()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) * 1e3 / (reps * ncopies)


out = {}
for name, mode, nimg, h, c0, c1, co in SHAPES:
    taps = 9 if mode else 1
    wbytes = co * taps * (c0 + c1) * 2
    ncopies = max(2, min(12, (160 << 20) // wbytes + 1))
    ws = [(torch.randn(co, taps * (c0 + c1), device="cuda") * 0.02).half() for _ in range(ncopies)]
    bias = torch.randn(nimg, co, device="cuda")
    if mode:
        x0 = torch.randn(nimg, h, h, c0, device="cuda").half()
        x1 = torch.randn(nimg, h, h, c1, device="cuda").half() if c1 else None
        res = torch.randn(nimg, h, h, co, device="cuda").half()
    else:
        x0 = torch.randn(nimg * h * h, c0, device="cuda").half()
        x1 = None
        res = torch.randn(nimg * h * h, co, device="cuda").half()
    kind = name.split("_")[0].rstrip("0123456789")  # qkv: no bias / residual; geglu: GEGLU epilogue, no residual
    if kind in ("qkv", "geglu"):
        res = None
    if kind == "qkv":
        bias = None
    rows = {}
    for cluster in (1, 0):
        os.environ["B200SD_CLUSTER_SPLITK"] = str(cluster)
        splits = [2, 4, 8] if cluster else [1, 2, 3, 4, 6, 8, 12, 16, 24, 32]
        cands = [(0, 0)] + [(bn, s) for bn in BNS for s in splits]
        for bn, s in cands:
            def fn(i, bn=bn, s=s):
                if mode:
                    return L.conv3x3(x0, ws[i], bias, res, x1=x1, bias_rows=h * h, block_n=bn, split_k=s)
                return L.linear(x0, ws[i], bias, res, bias_rows=0 if kind == "geglu" else h * h, block_n=bn, split_k=s,
                                static_w=True, geglu=kind == "geglu")
            try:
                us = time_graph(fn, ncopies)
            except Exception as e:  # candidate not realisable for this shape
                continue
            rows[f"{'C' if cluster else 'W'}:{bn}:{s}"] = round(us, 2)
    best = sorted((v, k) for k, v in rows.items() if not k.endswith(":0:0"))[:6]
    out[name] = {"auto_cluster": rows.get("C:0:0"), "auto_ws": rows.get("W:0:0"), "best": best}
    print(name, json.dumps(out[name]), flush=True)
    out[name]["rows"] = rows  # every candidate, for refitting the cost model
    L._tiled_cache.clear()
    del ws
    torch.cuda.empty_cache()
json.dump(out, open(sys.argv[1] if len(sys.argv) > 1 else "gemm_shapes.json", "w"), indent=1)
