"""Cost of grouping results by document (NOT the bench.py metric): search_device_masked (top-10 pages) against
search_docs_device (top-10 documents) on one bf16 corpus of 65 536 pages x 1024 patch rows (bench.py's synthetic shard),
and the selection alone (b200ms_topk against b200ms_topk_docs on one score matrix from b200ms_score).

Shapes: 1 and 32 queries of 32 tokens, k = 10, per_doc 1 and 4, over three document layouts: one page per document, 16
pages per document, and one document holding every page (every page's key lands on one word per query).  Every call is timed
with CUDA events on the current stream, p50 / p95 over --reps calls after --warmup.  Prints the card name and power limit
read in the same run, then one JSON line.

  python tools/bench_grouped.py [--pages 65536] [--reps 50] [--warmup 5]
"""
import argparse
import ctypes
import json
import os
import subprocess
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

import numpy as np  # noqa: E402
import torch  # noqa: E402

import bench  # noqa: E402
from morphik_core_b200 import _native as nat  # noqa: E402
from morphik_core_b200.index import MaxSimIndex  # noqa: E402

ap = argparse.ArgumentParser()
ap.add_argument("--pages", type=int, default=65536)
ap.add_argument("--reps", type=int, default=50)
ap.add_argument("--warmup", type=int, default=5)
args = ap.parse_args()

if not torch.cuda.is_available():
    sys.exit("bench_grouped.py needs a CUDA device (H100); nothing is measured without one")
dev = torch.device("cuda", 0)
card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,enforced.power.limit,power.max_limit,clocks.max.sm",
                       "--format=csv,noheader", "-i", "0"], capture_output=True, text=True).stdout.strip()
print(f"[bench_grouped] card: {card}", flush=True)

n = args.pages
q_host = bench.make_queries(32)
packed, _ = bench.build_shard(n, dev, 1234, q_host, planted_per_query=10)
idx = MaxSimIndex(dtype="bf16")
idx.adopt_packed(packed, [bench.P_PATCH] * n)
idx._attach()
q_dev = q_host.to(dev)
layouts = {"page_per_doc": (torch.arange(n, dtype=torch.int32, device=dev), n),
           "16_pages_per_doc": (torch.arange(n, dtype=torch.int32, device=dev) // 16, n // 16),
           "one_doc": (torch.zeros(n, dtype=torch.int32, device=dev), 1)}


def timed(fn):
    for _ in range(args.warmup):
        fn()
    ev = [(torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)) for _ in range(args.reps)]
    for a, b in ev:
        a.record()
        fn()
        b.record()
    torch.cuda.synchronize()
    ms = [a.elapsed_time(b) for a, b in ev]
    return round(float(np.median(ms)), 4), round(float(np.percentile(ms, 95)), 4)


def vp(t):
    return ctypes.c_void_p(t.data_ptr())


line = {"workload": f"{n} pages x {bench.P_PATCH} patches bf16, {bench.T_TOK}-token queries, k=10", "card": card}
k = 10
for n_q in (1, 32):
    lens = [bench.T_TOK] * n_q
    src = q_dev[: n_q * bench.T_TOK].contiguous()
    mi = torch.full((n_q,), -1, dtype=torch.int32, device=dev)
    full = torch.zeros((1, (n + 31) // 32), dtype=torch.int32, device=dev)
    line[f"q{n_q}_flat_ms"] = timed(lambda: idx.search_device(src, lens, k, allow_mask_dev=full, mask_index_dev=mi))
    gs, goff, _, _ = idx.score_groups([src[i * bench.T_TOK:(i + 1) * bench.T_TOK] for i in range(n_q)])
    goff_c = nat.i32_array(goff)
    ts = torch.empty((n_q, k * 4), dtype=torch.float32, device=dev)
    ti = torch.empty((n_q, k * 4), dtype=torch.int64, device=dev)
    tc = torch.empty((n_q, k), dtype=torch.int32, device=dev)
    dc = torch.empty((n_q,), dtype=torch.int32, device=dev)
    stream = ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)

    def flat_sel():
        idx.h.check(nat.lib.b200ms_topk(idx.h.ptr, vp(gs), nat.F32, n, gs.shape[1], goff_c, n_q, None, k, ctypes.c_float(1), 0,
                                        vp(ts), vp(ti), vp(dc), stream), "b200ms_topk")

    line[f"q{n_q}_select_flat_ms"] = timed(flat_sel)
    for name, (pd, n_docs) in layouts.items():
        for per_doc in (1, 4):
            line[f"q{n_q}_{name}_m{per_doc}_docs_ms"] = timed(
                lambda: idx.search_docs_device(src, lens, k, per_doc, pd, n_docs, allow_mask_dev=full, mask_index_dev=mi))

            def docs_sel():
                idx.h.check(nat.lib.b200ms_topk_docs(idx.h.ptr, vp(gs), nat.F32, n, gs.shape[1], goff_c, n_q, None, vp(pd), n_docs,
                                                     k, per_doc, ctypes.c_float(1), 0, vp(ts), vp(ti), vp(tc), vp(dc), stream),
                            "b200ms_topk_docs")

            line[f"q{n_q}_{name}_m{per_doc}_select_docs_ms"] = timed(docs_sel)
    # the identity layout with per_doc 1 is the flat top-k: same ids
    flat = idx.search_device(src, lens, k)[1]
    grouped = idx.search_docs_device(src, lens, k, 1, *layouts["page_per_doc"])[1][:, :, 0]
    assert torch.equal(flat, grouped)
print(json.dumps(line), flush=True)
