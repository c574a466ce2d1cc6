"""Timing of the scoring kernels, CUDA events, outside any profiler (developer aid; not a bench.py leg).

  python tools/time_scan.py [--pages 65536] [--dtypes bf16,int8,fp8] [--b1-groups 1,2,3,4,8]

Prints one JSON line: the GPU's name and power limit, scoring-kernel ms and GB/s for ONE 32-token query and ms for a
32-query batch per dtype, and with --b1-groups the 1-bit full-scan ms on the POPC kernel (b1_tensor 0) and on the wgmma
kernel (b1_tensor 1) for each number of 32-token query groups -- the measurement behind the b1_tensor = 2 crossover.
"""
import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

ap = argparse.ArgumentParser()
ap.add_argument("--pages", type=int, default=65536)
ap.add_argument("--dtypes", default="bf16,int8,fp8")
ap.add_argument("--b1-groups", default="", help="comma-separated query-group counts for the 1-bit POPC / wgmma comparison")
ap.add_argument("--steps", type=int, default=30)
args = ap.parse_args()

import torch  # noqa: E402

import bench  # noqa: E402
from morphik_core_b200.index import MaxSimIndex  # noqa: E402

dev = torch.device("cuda", 0)
q_host = bench.make_queries(32)
packed, _ = bench.build_shard(args.pages, dev, 1234, q_host)
q_dev = q_host.to(dev)
gpu = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                     text=True).stdout.strip()
out = {"gpu": gpu, "pages": args.pages}
for dt in [d for d in args.dtypes.split(",") if d]:
    if dt == "bf16":
        idx = MaxSimIndex(device=0, dtype="bf16")
        idx.adopt_packed(packed, [bench.P_PATCH] * args.pages)
    else:
        idx = bench.quantised_subshard(packed, args.pages, dt, 0)
    rb = idx.row_bytes
    _, one = bench.time_search(idx, q_dev[:32], [32], 10, args.steps, 5)
    _, b32 = bench.time_search(idx, q_dev, [32] * 32, 10, args.steps, 3)
    out[dt] = {"one_query_ms": round(one, 4), "one_query_gbs": round(args.pages * bench.P_PATCH * rb / one / 1e6, 1),
               "batch32_ms": round(b32, 4)}
    idx.close()
if args.b1_groups:
    idx = bench.quantised_subshard(packed, args.pages, "binary", 0)
    b1 = {}
    for ng in [int(x) for x in args.b1_groups.split(",")]:
        row = {}
        for path, name in ((0, "popc_ms"), (1, "wgmma_ms")):
            idx.set_option("b1_tensor", path)
            _, ms = bench.time_search(idx, q_dev[: ng * 32].contiguous(), [32] * ng, 10, args.steps, 3)
            row[name] = round(ms, 3)
        b1[ng] = row
    out["binary_full_scan_by_groups"] = b1
    idx.close()
print(json.dumps(out))
