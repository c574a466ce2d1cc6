"""Latency probe of MaxSimIndex.explain (NOT the bench.py metric) next to the search that produced the explained pages, on one
bf16 corpus of 65 536 pages x 1024 patch rows (bench.py's synthetic shard).  Two shapes:
  * 1 query x top-10, with the full token x row similarity map (what a UI highlighting the matched regions asks for);
  * 32 queries x top-100, token scores and best rows only (ranking diagnostics over a batch).
Explain and search are timed as calls from device-resident query rows to device-resident results, host clock around a device
synchronise, p50 / p95 over --reps calls after --warmup.  Prints the card name and power limit, then one JSON line.

  python tools/bench_explain.py [--pages 65536] [--reps 50] [--warmup 5]
"""
import argparse
import json
import os
import subprocess
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

import numpy as np  # noqa: E402
import torch  # noqa: E402

import bench  # noqa: E402
from morphik_core_b200.index import MaxSimIndex  # noqa: E402

ap = argparse.ArgumentParser()
ap.add_argument("--pages", type=int, default=65536)
ap.add_argument("--reps", type=int, default=50)
ap.add_argument("--warmup", type=int, default=5)
args = ap.parse_args()

if not torch.cuda.is_available():
    sys.exit("bench_explain.py needs a CUDA device (H100); nothing is measured without one")
dev = torch.device("cuda", 0)
card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,enforced.power.limit,power.max_limit,clocks.max.sm",
                       "--format=csv,noheader", "-i", "0"], capture_output=True, text=True).stdout.strip()
print(f"[bench_explain] card: {card}", flush=True)

q_host = bench.make_queries(32)
packed, _ = bench.build_shard(args.pages, dev, 1234, q_host, planted_per_query=10)
idx = MaxSimIndex(dtype="bf16")
idx.adopt_packed(packed, [bench.P_PATCH] * args.pages)
idx._attach()
q_dev = q_host.to(dev)
queries = [q_dev[i * bench.T_TOK:(i + 1) * bench.T_TOK] for i in range(32)]


def timed(fn):
    for _ in range(args.warmup):
        fn()
    torch.cuda.synchronize()
    ms = []
    for _ in range(args.reps):
        t0 = time.perf_counter()
        fn()
        torch.cuda.synchronize()
        ms.append((time.perf_counter() - t0) * 1e3)
    return float(np.median(ms)), float(np.percentile(ms, 95))


line = {"workload": f"{args.pages} pages x {bench.P_PATCH} patches bf16, {bench.T_TOK}-token queries", "card": card}
for name, n_q, k, map_rows in (("q1_top10_map", 1, 10, bench.P_PATCH), ("q32_top100", 32, 100, 0)):
    lens = [bench.T_TOK] * n_q
    src = q_dev[: n_q * bench.T_TOK].contiguous()
    ts, ti, tc = idx.search_device(src, lens, k)
    torch.cuda.synchronize()
    assert int(tc.min()) == k
    sp50, sp95 = timed(lambda: idx.search_device(src, lens, k))
    ep50, ep95 = timed(lambda: idx.explain(queries[:n_q], ti, map_rows))
    tok, _, _ = idx.explain(queries[:n_q], ti, map_rows)
    dev_sum = (tok.double().sum(dim=2) - ts.double()).abs().max().item()  # explanation adds up to the search's scores
    line.update({f"{name}_search_p50_ms": sp50, f"{name}_search_p95_ms": sp95, f"{name}_explain_p50_ms": ep50,
                 f"{name}_explain_p95_ms": ep95, f"{name}_max_abs_sum_minus_score": dev_sum,
                 f"{name}_explain_tflop": 2.0 * n_q * k * bench.P_PATCH * bench.T_TOK * bench.DIM / 1e12})
print(json.dumps(line), flush=True)
