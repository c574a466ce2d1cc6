"""Latency probe of relevance feedback (MaxSimIndex.search_examples, TwoStageIndex.search_examples_device) -- NOT the
bench.py metric -- on bench.py's topic corpus: 65 536 pages x 1024 patch rows, bf16 and int8, k = 10.

Workload: one request of a 32-token query and 2 liked + 1 disliked stored pages (1024 rows each), weights +1/3 and -1.
  * exhaustive (HBM full scan) and FDE two-stage with 75 candidates per positive: the whole call, CUDA events around it,
    p50 / p95;
  * the device time of the fusion kernel and (two-stage) the union kernel, from torch.profiler, and their share of the call.
Prints the card name and power limit, then one JSON line.

  python tools/bench_examples.py [--pages 65536] [--reps 10] [--warmup 2] [--dtypes bf16,int8]
"""
import argparse
import json
import os
import subprocess
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

import numpy as np  # noqa: E402
import torch  # noqa: E402
from torch.profiler import ProfilerActivity, profile  # noqa: E402

import bench  # noqa: E402
from morphik_core_b200.fde import TwoStageIndex  # noqa: E402

ap = argparse.ArgumentParser()
ap.add_argument("--pages", type=int, default=65536)
ap.add_argument("--reps", type=int, default=10)
ap.add_argument("--warmup", type=int, default=2)
ap.add_argument("--dtypes", default="bf16,int8")
args = ap.parse_args()

if not torch.cuda.is_available():
    sys.exit("bench_examples.py needs a CUDA device (H100); nothing is measured without one")
dev = torch.device("cuda", 0)
card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                      capture_output=True, text=True).stdout.strip()
print(f"[bench_examples] card: {card}", flush=True)

ROWS = bench.P_PATCH
N_CAND = 75
anchors = bench.topic_anchors(dev)
q_host, _ = bench.make_topic_queries(8, anchors)
packed, _ = bench.build_shard(args.pages, dev, seed=1234, q_host=q_host, topic_pages=args.pages // 2, anchors=anchors)
rng = np.random.default_rng(7)
PAGES = [int(p) for p in rng.choice(args.pages, size=3, replace=False)]  # 2 liked, 1 disliked
QUERY = q_host[:bench.T_TOK].numpy()
EX_REQ, WEIGHTS = [0, 0, 0, 0], [1 / 3, 1 / 3, 1 / 3, -1.0]


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


def kernel_ms(fn, names):
    """Mean device time per call of the kernels whose name contains each of `names` (torch.profiler, CUDA activity)."""
    reps = 3
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(reps):
            fn()
        torch.cuda.synchronize()
    out = {}
    for n in names:
        us = sum(e.device_time_total for e in prof.key_averages() if n in e.key)
        out[n] = round(us / reps / 1e3, 4)
    return out


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
    q_dev = torch.from_numpy(QUERY).to(dev)
    calls = {"exhaustive": lambda: idx.search_examples(q_dev, [len(QUERY)], PAGES, EX_REQ, WEIGHTS, 1, 10),
             f"fde_{N_CAND}": lambda: two.search_examples_device([QUERY], PAGES, EX_REQ, WEIGHTS, 1, 10, n_candidates=N_CAND)}
    for mode, fn in calls.items():
        call = timed(fn)
        kern = kernel_ms(fn, ["fuse_examples_kernel", "union_candidates_kernel"])
        p50 = float(np.median(call))
        row = {"dtype": dtype, "mode": mode, "call": pct(call), "fuse_kernel_ms": kern["fuse_examples_kernel"],
               "fuse_share_pct": round(100 * kern["fuse_examples_kernel"] / p50, 3)}
        if mode != "exhaustive":
            row["union_kernel_ms"] = kern["union_candidates_kernel"]
        print(f"[bench_examples] {json.dumps(row)}", flush=True)
        results.append(row)
    if dtype != "bf16":
        del idx, two
        torch.cuda.empty_cache()

print(json.dumps({"workload": f"{args.pages} pages x {ROWS} patches; a {bench.T_TOK}-token query + 2 liked and 1 disliked "
                              f"{ROWS}-row pages, k 10", "card": card, "results": results}))
