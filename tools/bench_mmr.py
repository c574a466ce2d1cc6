"""Latency probe of maximal marginal relevance (MaxSimIndex.mmr, B200MultiVectorStore.query_similar_mmr) -- NOT the bench.py
metric -- on bench.py's topic corpus: 65 536 pages x 1024 patch rows, bf16 and int8.

For fetch_k in {20, 100, 1000} and k in {5, 10, 50} (k <= fetch_k), over topic queries:
  * the MMR call alone (device-resident candidate lists from a search, CUDA events around the call), p50 / p95;
  * the round kernel's achieved TFLOP/s: its device time from torch.profiler over the pair count x 1024^2 x 256 FLOP (every
    live candidate against every pick but the last; 2 x 128 multiply-adds per row pair);
  * query_similar_mmr against query_similar on a store over the same index (host clock around each synchronous call), p50 / p95.
Prints the card name and power limit, then one JSON line.

  python tools/bench_mmr.py [--pages 65536] [--reps 20] [--warmup 3] [--dtypes bf16,int8]
"""
import argparse
import asyncio
import json
import os
import subprocess
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

import numpy as np  # noqa: E402
import torch  # noqa: E402

import bench  # noqa: E402
from morphik_core_b200.catalog import PageRecord  # noqa: E402
from morphik_core_b200.index import MaxSimIndex  # noqa: E402
from morphik_core_b200.store import B200MultiVectorStore  # noqa: E402

ap = argparse.ArgumentParser()
ap.add_argument("--pages", type=int, default=65536)
ap.add_argument("--reps", type=int, default=20)
ap.add_argument("--warmup", type=int, default=3)
ap.add_argument("--dtypes", default="bf16,int8")
args = ap.parse_args()

if not torch.cuda.is_available():
    sys.exit("bench_mmr.py needs a CUDA device (H100); nothing is measured without one")
dev = torch.device("cuda", 0)
card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                      capture_output=True, text=True).stdout.strip()
print(f"[bench_mmr] card: {card}", flush=True)

FETCH, KS = (20, 100, 1000), (5, 10, 50)
ROWS = bench.P_PATCH
anchors = bench.topic_anchors(dev)
q_host, _ = bench.make_topic_queries(8, anchors)
topic_pages = args.pages // 2
packed, _ = bench.build_shard(args.pages, dev, seed=1234, q_host=q_host, topic_pages=topic_pages, anchors=anchors)
queries = [q_host[i * bench.T_TOK:(i + 1) * bench.T_TOK].numpy() for i in range(8)]


def pct(ms):
    return {"p50_ms": round(float(np.median(ms)), 4), "p95_ms": round(float(np.percentile(ms, 95)), 4)}


def event_ms(fn):
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    fn()
    b.record()
    b.synchronize()
    return a.elapsed_time(b)


def round_kernel_ms(fn, reps=3):
    from torch.profiler import ProfilerActivity, profile

    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(reps):
            fn()
        torch.cuda.synchronize()
    us = sum(getattr(e, "device_time_total", getattr(e, "cuda_time_total", 0)) for e in prof.key_averages()
             if "mmr_round" in e.key)
    return us / 1e3 / reps


results = []
for dtype in args.dtypes.split(","):
    if dtype == "bf16":
        idx = MaxSimIndex(dtype="bf16")
        idx.adopt_packed(packed, [ROWS] * args.pages)
    else:
        idx = bench.quantised_subshard(packed, args.pages, dtype, 0)
    idx._attach()
    store = B200MultiVectorStore(mode=dtype, index=idx, auto_initialize=False, coalesce_queries=False)
    for p in range(args.pages):
        store.catalog.add(PageRecord(f"doc{p}", 0, "", {}, None, ROWS))
    for fetch_k in FETCH:
        # candidate lists: the search's own top fetch_k of every query
        lists = []
        for q in queries:
            ts, ti, tc = idx.search_device(torch.from_numpy(q).to(dev), [bench.T_TOK], fetch_k)
            lists.append((ti, ts))
        torch.cuda.synchronize()
        for k in KS:
            if k > fetch_k:
                continue

            def one(i):
                ti, ts = lists[i % len(lists)]
                return idx.mmr(ti, ts, [bench.T_TOK], k, 0.5)

            for i in range(args.warmup):
                one(i)
            call = [event_ms(lambda i=i: one(i)) for i in range(args.reps)]
            rk_ms = round_kernel_ms(lambda: one(0))
            pairs = sum(fetch_k - i for i in range(1, min(k, fetch_k)))
            flop = pairs * ROWS * ROWS * 2 * bench.DIM

            def store_ms(fn, n):
                out = []
                for i in range(args.warmup + n):
                    t0 = time.perf_counter()
                    asyncio.run(fn(queries[i % len(queries)]))
                    if i >= args.warmup:
                        out.append((time.perf_counter() - t0) * 1e3)
                return out

            mmr_store = store_ms(lambda q: store.query_similar_mmr(q, k=k, fetch_k=fetch_k, lambda_mult=0.5), args.reps)
            flat_store = store_ms(lambda q: store.query_similar(q, k=k), args.reps)
            row = {"dtype": dtype, "fetch_k": fetch_k, "k": k, "mmr_call": pct(call),
                   "round_kernel_ms": round(rk_ms, 4), "round_pairs": pairs,
                   "round_tflops": round(flop / (rk_ms * 1e-3) / 1e12, 1) if rk_ms > 0 else None,
                   "query_similar_mmr": pct(mmr_store), "query_similar": pct(flat_store)}
            print(f"[bench_mmr] {json.dumps(row)}", flush=True)
            results.append(row)
    store.close()
    del idx, store
    torch.cuda.empty_cache()

print(json.dumps({"workload": f"{args.pages} pages x {ROWS} patches, {bench.T_TOK}-token topic queries, lambda_mult 0.5",
                  "card": card, "results": results}))
