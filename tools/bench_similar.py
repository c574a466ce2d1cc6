"""Latency probe of searching with stored pages as the queries (MaxSimIndex.search_pages, TwoStageIndex.search_pages) --
NOT the bench.py metric -- on bench.py's topic corpus: 65 536 pages x 1024 patch rows, bf16 and int8.

For batches of 1 and 16 source pages of 1024 rows each:
  * exhaustive (HBM full scan) and FDE two-stage with 75 and 1000 candidates: the whole call, CUDA events around it, p50 / p95;
  * exhaustive only: the scan kernels' device time (b200ms_score_times_ms, the events around the scoring launches) and
    their achieved TFLOP/s over n_src x pages x 1024 x 1024 x 256 FLOP (2 x 128 multiply-adds per row pair; int8: TOPS).
Prints the card name and power limit, then one JSON line.

  python tools/bench_similar.py [--pages 65536] [--reps 10] [--warmup 2] [--dtypes bf16,int8]
"""
import argparse
import json
import os
import subprocess
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

import numpy as np  # noqa: E402
import torch  # noqa: E402

import bench  # noqa: E402
from morphik_core_b200.fde import TwoStageIndex  # noqa: E402
from morphik_core_b200.index import MaxSimIndex  # noqa: E402

ap = argparse.ArgumentParser()
ap.add_argument("--pages", type=int, default=65536)
ap.add_argument("--reps", type=int, default=10)
ap.add_argument("--warmup", type=int, default=2)
ap.add_argument("--dtypes", default="bf16,int8")
args = ap.parse_args()

if not torch.cuda.is_available():
    sys.exit("bench_similar.py needs a CUDA device (H100); nothing is measured without one")
dev = torch.device("cuda", 0)
card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                      capture_output=True, text=True).stdout.strip()
print(f"[bench_similar] card: {card}", flush=True)

ROWS = bench.P_PATCH
BATCHES = (1, 16)
CANDIDATES = (75, 1000)
anchors = bench.topic_anchors(dev)
q_host, _ = bench.make_topic_queries(8, anchors)
packed, _ = bench.build_shard(args.pages, dev, seed=1234, q_host=q_host, topic_pages=args.pages // 2, anchors=anchors)
rng = np.random.default_rng(7)
SOURCES = [int(p) for p in rng.choice(args.pages, size=max(BATCHES), replace=False)]


def pct(ms):
    return {"p50_ms": round(float(np.median(ms)), 3), "p95_ms": round(float(np.percentile(ms, 95)), 3)}


def event_ms(fn):
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    fn()
    b.record()
    b.synchronize()
    return a.elapsed_time(b)


def timed(fn):
    for _ in range(args.warmup):
        fn()
    return [event_ms(fn) for _ in range(args.reps)]


fde_bf16 = TwoStageIndex(dtype="bf16")
fde_bf16.adopt_packed(packed, [ROWS] * args.pages)
results = []
for dtype in args.dtypes.split(","):
    if dtype == "bf16":
        idx, two = fde_bf16.index, fde_bf16
    else:
        idx = bench.quantised_subshard(packed, args.pages, dtype, 0)
        two = TwoStageIndex(index=idx)  # the same FDE rows: they come from the float pages, not the corpus dtype
        two.append_fde_rows(*fde_bf16.fde_rows())
    idx._attach()
    for n_src in BATCHES:
        src = SOURCES[:n_src]
        call = timed(lambda: idx.search_pages(src, 10))
        scan_ms = float(np.median(idx.score_times_ms(args.reps)))
        flop = n_src * args.pages * ROWS * ROWS * 2 * bench.DIM
        row = {"dtype": dtype, "n_src": n_src, "src_rows": ROWS, "mode": "exhaustive", "call": pct(call),
               "scan_kernel_ms": round(scan_ms, 3), "scan_tflops": round(flop / (scan_ms * 1e-3) / 1e12, 1)}
        print(f"[bench_similar] {json.dumps(row)}", flush=True)
        results.append(row)
        for n_cand in CANDIDATES:
            call = timed(lambda: two.search_pages_device(src, 10, n_candidates=n_cand))
            row = {"dtype": dtype, "n_src": n_src, "src_rows": ROWS, "mode": f"fde_{n_cand}", "call": pct(call)}
            print(f"[bench_similar] {json.dumps(row)}", flush=True)
            results.append(row)
    if dtype != "bf16":
        del idx, two
        torch.cuda.empty_cache()

print(json.dumps({"workload": f"{args.pages} pages x {ROWS} patches, {ROWS}-row source pages, k 10", "card": card,
                  "results": results}))
