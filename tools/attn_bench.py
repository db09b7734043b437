"""Times the attention kernel on every attention shape the flagship (SD-2.1-base 512x512, batch 2), the SDXL-768 config
and SD-1.5 (512x512, batch 2: 8 heads of head dim 40 / 80 / 160) launch: self-attention over fused q|k|v views and
cross-attention against 77 text tokens.  Each shape: 50 back-to-back launches captured in one CUDA graph (so host-side
launch cost is not timed), replayed between CUDA events, best of 5; prints microseconds per launch and TFLOP/s
(4 * B * H * Sq * Sk * d FLOP) per shape.  The schedule is the one the models get (stream-K where it pays);
B200SD_ATTN_STREAMK=0 in the environment times whole-tile scheduling instead.  --d 40 (etc.) times one head dim only.

--dump DIR writes each shape's output for seeded inputs as DIR/<name>.npy (float32), so two builds can be compared."""
import argparse
import json
import os
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import b200sd  # noqa: E402,F401
from b200sd import lib  # noqa: E402

# (kind, batch, heads, sq, sk, d)
SHAPES = [
    ("self", 2, 5, 4096, 4096, 64), ("self", 2, 10, 1024, 1024, 64), ("self", 2, 20, 256, 256, 64),
    ("self", 2, 20, 64, 64, 64),
    ("cross", 2, 5, 4096, 77, 64), ("cross", 2, 10, 1024, 77, 64), ("cross", 2, 20, 256, 77, 64),
    ("cross", 2, 20, 64, 77, 64),
    ("self", 2, 10, 2304, 2304, 64), ("self", 2, 20, 576, 576, 64),  # SDXL-768
    # SD-1.5
    ("self", 2, 8, 4096, 4096, 40), ("self", 2, 8, 1024, 1024, 80), ("self", 2, 8, 256, 256, 160),
    ("self", 2, 8, 64, 64, 160),
    ("cross", 2, 8, 4096, 77, 40), ("cross", 2, 8, 1024, 77, 80), ("cross", 2, 8, 256, 77, 160),
    ("cross", 2, 8, 64, 77, 160),
]


def timed(fn, n=50, reps=5):
    """Best-of-reps time per launch of fn, with n launches captured in one CUDA graph."""
    stream = torch.cuda.Stream()
    stream.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(stream):
        fn()  # the first launch sets kernel attributes and allocates the workspace outside the capture
    torch.cuda.current_stream().wait_stream(stream)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        for _ in range(n):
            fn()
    graph.replay()
    best = 1e9
    for _ in range(reps):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        torch.cuda.synchronize()
        a.record()
        graph.replay()
        b.record()
        torch.cuda.synchronize()
        best = min(best, a.elapsed_time(b) / n * 1e3)
    return best


def operands(kind, batch, heads, sq, sk, d, seed):
    """q, k, v as the UNet passes them: strided views of one fused q|k|v (self) or q plus a fused k|v (cross)."""
    c = heads * d
    g = torch.Generator().manual_seed(seed)
    if kind == "self":
        qkv = torch.randn(batch * sq, 3 * c, generator=g).half().cuda()
        return qkv[:, :c], qkv[:, c:2 * c], qkv[:, 2 * c:]
    q = torch.randn(batch * sq, c, generator=g).half().cuda()
    kv = torch.randn(batch * sk, 2 * c, generator=g).half().cuda()
    return q, kv[:, :c], kv[:, c:]


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n")[0])
    ap.add_argument("--dump", metavar="DIR", default=None, help="write each shape's output as DIR/<name>.npy")
    ap.add_argument("--d", type=int, default=None, help="time only the shapes of this head dim")
    args = ap.parse_args()
    if args.dump:
        os.makedirs(args.dump, exist_ok=True)
    for i, (kind, batch, heads, sq, sk, d) in enumerate(SHAPES):
        if args.d is not None and d != args.d:
            continue
        q, k, v = operands(kind, batch, heads, sq, sk, d, seed=1234 + i)
        out = torch.empty(batch * sq, heads * d, dtype=torch.float16, device="cuda")
        name = f"{kind}_{batch}x{heads}x{sq}x{sk}" + ("" if d == 64 else f"_d{d}")
        lib.attention(q, k, v, batch, heads, sq, sk, d=d, out=out)
        if args.dump:
            torch.cuda.synchronize()
            np.save(os.path.join(args.dump, name + ".npy"), out.float().cpu().numpy())
        us = timed(lambda: lib.attention(q, k, v, batch, heads, sq, sk, d=d, out=out))
        tflops = 4.0 * batch * heads * sq * sk * d / us * 1e-6
        print(json.dumps({"shape": name, "us": round(us, 2), "tflops": round(tflops, 1)}), flush=True)


if __name__ == "__main__":
    main()
