"""ncu launch list with dram__bytes_read.sum / dram__bytes_write.sum / gpu__time_duration.sum (cold caches: ncu flushes
L2 before every kernel) -> a JSON file: DRAM bytes per launch of the GEMM / convolution kernels and per kernel."""
import collections
import csv
import io
import json
import sys


def main(path, out):
    lines = open(path).read().splitlines()
    start = next(i for i, l in enumerate(lines) if l.startswith('"ID"'))
    rows = list(csv.DictReader(io.StringIO("\n".join(lines[start:]))))
    per = collections.defaultdict(lambda: {"launches": set(), "read_bytes": 0.0, "write_bytes": 0.0, "us": 0.0})
    scale = {"byte": 1.0, "Kbyte": 1e3, "Mbyte": 1e6, "Gbyte": 1e9, "ns": 1e-3, "us": 1.0, "usecond": 1.0, "nsecond": 1e-3,
             "msecond": 1e3, "ms": 1e3}
    for r in rows:
        name = r["Kernel Name"].split("(")[0].replace("void ", "")
        name = name.split("<")[0] if name.startswith("b200sd::") else name
        name = name.replace("b200sd::", "")
        v = float(r["Metric Value"].replace(",", "")) * scale[r["Metric Unit"]]
        e = per[name]
        e["launches"].add(r["ID"])
        if r["Metric Name"] == "dram__bytes_read.sum":
            e["read_bytes"] += v
        elif r["Metric Name"] == "dram__bytes_write.sum":
            e["write_bytes"] += v
        else:
            e["us"] += v
    for e in per.values():
        e["launches"] = len(e["launches"])
    gemm = [e for k, e in per.items() if k.startswith(("wgmma_gemm", "halo_conv", "splitk_reduce"))]
    n = sum(e["launches"] for k, e in per.items() if k.startswith(("wgmma_gemm", "halo_conv")))
    tot = sum(e["read_bytes"] + e["write_bytes"] for e in gemm)
    doc = {"source": f"{path} (ncu dram__bytes_read.sum + dram__bytes_write.sum of ONE bench.py iteration, "
                     "`bench.py --profile-step`; L2 flushed before every kernel by ncu, so activations that stay in L2 "
                     "during a real step are counted as DRAM reads here: an upper bound)",
           "kernel": "wgmma_gemm_kernel (all variants) + splitk_reduce_kernel", "launches": n,
           "dram_bytes_per_forward": tot, "dram_bytes_per_launch": tot / max(n, 1),
           "algorithmic_weight_bytes_per_forward": 1.73e9, "per_kernel": dict(sorted(per.items()))}
    json.dump(doc, open(out, "w"), indent=1)
    print(out, n, "GEMM launches,", round(tot / 1e9, 3), "GB DRAM per forward")


if __name__ == "__main__":
    main(sys.argv[1], sys.argv[2])
