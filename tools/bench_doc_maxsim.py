"""Latency probe of document-level MaxSim (MaxSimIndex.search_doc_maxsim_device) -- NOT the bench.py metric -- next to the
best-page document search (search_docs_device), on bench.py's topic corpus: 65 536 pages x 1024 patch rows, 16 pages per
document (4096 documents), bf16 and int8, k = 10, per_doc = 4.

For 1 and 32 queries of bench.py's 32 tokens:
  * p50 / p95 of both calls, CUDA events around each call, the two alternated in one process;
  * the device time of the document-mode scan and of the document kernels (sum, selection, evidence), and of the page
    scan of search_docs_device, from torch.profiler in a separate pass;
  * the share of identical top-1 documents between the two calls (they rank by different scores: not a check).
Prints the card name and power limit, then one JSON line.

  python tools/bench_doc_maxsim.py [--pages 65536] [--reps 20] [--warmup 3] [--dtypes bf16,int8]
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
from morphik_core_b200.index import MaxSimIndex  # noqa: E402

ap = argparse.ArgumentParser()
ap.add_argument("--pages", type=int, default=65536)
ap.add_argument("--reps", type=int, default=20)
ap.add_argument("--warmup", type=int, default=3)
ap.add_argument("--dtypes", default="bf16,int8")
args = ap.parse_args()

if not torch.cuda.is_available():
    sys.exit("bench_doc_maxsim.py needs a CUDA device (H100); nothing is measured without one")
dev = torch.device("cuda", 0)
card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                      capture_output=True, text=True).stdout.strip()
print(f"[bench_doc_maxsim] card: {card}", flush=True)

ROWS = bench.P_PATCH
PAGES_PER_DOC = 16
K, PER_DOC = 10, 4
anchors = bench.topic_anchors(dev)
q_host, _ = bench.make_topic_queries(32, anchors)
packed, _ = bench.build_shard(args.pages, dev, seed=1234, q_host=q_host, topic_pages=args.pages // 2, anchors=anchors)
N_DOCS = args.pages // PAGES_PER_DOC
PAGE_DOC = (torch.arange(args.pages, dtype=torch.int32, device=dev) // PAGES_PER_DOC).contiguous()
# kernels of each leg, by name fragment
DOC_SCAN, PAGE_SCAN = "maxsim_wgmma_doc_kernel", "maxsim_wgmma_kernel"
DOC_KERNELS = ["doc_sum_kernel", "doc_evidence_kernel", "topk"]


def pct(ms):
    return {"p50_ms": round(float(np.median(ms)), 3), "p95_ms": round(float(np.percentile(ms, 95)), 3)}


def event_ms(fn):
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    fn()
    b.record()
    b.synchronize()
    return a.elapsed_time(b)


def kernel_ms(fn, names):
    """Mean device time per call of the kernels whose name contains each of `names` (torch.profiler, CUDA activity)."""
    reps = 3
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(reps):
            fn()
        torch.cuda.synchronize()
    out = {}
    for n in names:
        us = sum(e.device_time_total for e in prof.key_averages()
                 if n in e.key and not (n == PAGE_SCAN and DOC_SCAN in e.key))
        out[n] = round(us / reps / 1e3, 4)
    return out


results = []
for dtype in args.dtypes.split(","):
    if dtype == "bf16":
        idx = MaxSimIndex(dtype="bf16")
        idx.adopt_packed(packed, [ROWS] * args.pages)
    else:
        idx = bench.quantised_subshard(packed, args.pages, dtype, 0)
    idx._attach()
    for n_q in (1, 32):
        q = q_host[:n_q * bench.T_TOK].to(dev).contiguous()
        lens = [bench.T_TOK] * n_q
        calls = {
            "doc_maxsim": lambda: idx.search_doc_maxsim_device(q, lens, K, PER_DOC, PAGE_DOC, N_DOCS),
            "search_docs": lambda: idx.search_docs_device(q, lens, K, PER_DOC, PAGE_DOC, N_DOCS),
        }
        for fn in calls.values():
            for _ in range(args.warmup):
                fn()
        times = {name: [] for name in calls}
        for _ in range(args.reps):  # alternated
            for name, fn in calls.items():
                times[name].append(event_ms(fn))
        dm = [t.cpu() for t in calls["doc_maxsim"]()]
        sd = [t.cpu() for t in calls["search_docs"]()]
        same_top1 = float((dm[1][:, 0] == sd[1][:, 0, 0] // PAGES_PER_DOC).float().mean())
        kd = kernel_ms(calls["doc_maxsim"], [DOC_SCAN] + DOC_KERNELS)
        kp = kernel_ms(calls["search_docs"], [PAGE_SCAN])
        row = {"dtype": dtype, "n_q": n_q, "doc_maxsim": pct(times["doc_maxsim"]), "search_docs": pct(times["search_docs"]),
               "p50_ratio": round(float(np.median(times["doc_maxsim"]) / np.median(times["search_docs"])), 4),
               "doc_scan_kernel_ms": kd[DOC_SCAN], "page_scan_kernel_ms": kp[PAGE_SCAN],
               "doc_sum_ms": kd["doc_sum_kernel"], "doc_evidence_ms": kd["doc_evidence_kernel"], "doc_topk_ms": kd["topk"],
               "same_top1_document": round(same_top1, 3)}
        print(f"[bench_doc_maxsim] {json.dumps(row)}", flush=True)
        results.append(row)
    del idx
    torch.cuda.empty_cache()

print(json.dumps({"workload": f"{args.pages} pages x {ROWS} patches, {PAGES_PER_DOC} pages per document, "
                              f"{bench.T_TOK}-token queries, k {K}, per_doc {PER_DOC}", "card": card, "results": results}))
