"""Filtered search: the masked search (scans only the allowed pages) against the scan of every page followed by a masked
top-k, CUDA events, outside any profiler (developer aid; not a bench.py leg).

  python tools/bench_filtered.py [--pages 65536] [--dtypes bf16,int8] [--reps 30] [--warmup 5]

Shard: --pages pages x 1024 rows x 128, 16 pages per document.  For one 32-token query and a batch of 32, and for masks of
whole documents drawn at random (100 / 50 / 10 / 1 / 0.1 % of the documents) plus one mask of single pages drawn at random
(10 %, the shortest runs a filter can have), it alternates in one process
  (a) search_device with the mask, and
  (b) b200ms_score over every page + b200ms_topk with the mask (what a masked search cost before it planned its scan),
and prints one JSON line: the GPU's name and power limit, per configuration the p50 of both in ms, the bytes (a) has to
read (padded rows of the allowed pages x row bytes) and the bytes/s that makes of (a)'s p50 (the whole call: pack, plan,
scan and top-k), and whether both returned the same bits.  Without a GPU it fails.
"""
import argparse
import ctypes
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

ap = argparse.ArgumentParser()
ap.add_argument("--pages", type=int, default=65536)
ap.add_argument("--dtypes", default="bf16,int8")
ap.add_argument("--reps", type=int, default=30)
ap.add_argument("--warmup", type=int, default=5)
ap.add_argument("--k", type=int, default=10)
args = ap.parse_args()

import numpy as np  # noqa: E402
import torch  # noqa: E402

import bench  # noqa: E402
from morphik_core_b200 import _native as nat  # noqa: E402
from morphik_core_b200.index import MaxSimIndex  # noqa: E402

if not torch.cuda.is_available():
    sys.exit("bench_filtered: no CUDA device (this measurement has no CPU form)")
dev = torch.device("cuda", 0)
PAGES_PER_DOC = 16
K = args.k
vp = lambda t: ctypes.c_void_p(t.data_ptr())  # noqa: E731


def masks_for(n_pages, rng):
    n_docs = n_pages // PAGES_PER_DOC
    out = {}
    for pct in (100, 50, 10, 1, 0.1):
        docs = np.zeros(n_docs, bool)
        docs[rng.choice(n_docs, size=max(1, round(n_docs * pct / 100)), replace=False)] = True
        allow = np.zeros(n_pages, bool)
        allow[: n_docs * PAGES_PER_DOC] = np.repeat(docs, PAGES_PER_DOC)
        out[f"documents_{pct}pct"] = allow
    out["random_pages_10pct"] = rng.random(n_pages) < 0.10
    return out


def p50(ms):
    return float(np.percentile(ms, 50))


def measure(idx, q_dev, q_lens, allow):
    """p50 ms of (a) and (b), alternated, and whether their outputs agree bit for bit."""
    n_q = len(q_lens)
    mask = torch.from_numpy(idx.mask_from_pages(allow).view(np.int32)).to(dev)
    out_a = tuple(torch.empty(s, dtype=d, device=dev) for s, d in (((n_q, K), torch.float32), ((n_q, K), torch.int64), ((n_q,), torch.int32)))
    out_b = tuple(torch.empty_like(t) for t in out_a)
    h = idx.h
    lens_c = nat.i32_array(q_lens)
    groups = int(nat.lib.b200ms_query_groups(lens_c, n_q))
    gp = max((groups + 3) // 4 * 4, 4)
    ld = (idx.n_pages + 31) // 32 * 32
    scores = torch.zeros((gp, ld), dtype=torch.float32 if idx.float_scores else torch.int32, device=dev)
    q_packed = torch.empty(gp * 32 * idx.row_bytes + 1024, dtype=torch.uint8, device=dev)
    q_packed = q_packed[(-q_packed.data_ptr()) % 1024:][: gp * 32 * idx.row_bytes]
    goff = (ctypes.c_int32 * (n_q + 1))()
    ng = ctypes.c_int(0)
    sdt = nat.F32 if idx.float_scores else nat.I32
    src_dtype = nat.BF16 if q_dev.dtype == torch.bfloat16 else nat.F32
    scale, i8 = ctypes.c_float(idx.score_scale), ctypes.c_float(idx.i8_scale)

    def run_a():
        idx.search_device(q_dev, q_lens, K, allow_mask_dev=mask, out=out_a)

    def run_b():
        s = idx._stream()
        h.check(nat.lib.b200ms_pack_queries(h.ptr, vp(q_dev), src_dtype, lens_c, n_q, vp(q_packed), idx.dtype, i8, goff,
                                            ctypes.byref(ng), s), "b200ms_pack_queries")
        h.check(nat.lib.b200ms_score(h.ptr, vp(q_packed), ng.value, lens_c, goff, n_q, vp(scores), ld, s), "b200ms_score")
        h.check(nat.lib.b200ms_topk(h.ptr, vp(scores), sdt, idx.n_pages, ld, goff, n_q, vp(mask), K, scale, 0, vp(out_b[0]),
                                    vp(out_b[1]), vp(out_b[2]), s), "b200ms_topk")

    ms = {"a": [], "b": []}
    for i in range(args.warmup + args.reps):
        for name, fn in (("a", run_a), ("b", run_b)):
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            fn()
            e1.record()
            e1.synchronize()
            if i >= args.warmup:
                ms[name].append(e0.elapsed_time(e1))
    same = all(torch.equal(a.view(torch.uint8), b.view(torch.uint8)) for a, b in zip(out_a, out_b))
    run_a()  # the plan of an (a) call is the last one the stats describe
    stats = idx.scan_stats()
    return p50(ms["a"]), p50(ms["b"]), same, stats


q_host = bench.make_queries(32)
packed, _ = bench.build_shard(args.pages, dev, 1234, q_host)
q_all = q_host.to(dev)
out = {"gpu": bench.gpu_name_and_power_limit(0), "pages": args.pages, "rows_per_page": bench.P_PATCH, "reps": args.reps,
       "results": []}
rng = np.random.default_rng(2026)
masks = masks_for(args.pages, rng)
for dt in [d for d in args.dtypes.split(",") if d]:
    if dt == "bf16":
        idx = MaxSimIndex(device=0, dtype="bf16")
        idx.adopt_packed(packed, [bench.P_PATCH] * args.pages)
    else:
        idx = bench.quantised_subshard(packed, args.pages, dt, 0)
    for n_q in (1, 32):
        q_dev, q_lens = q_all[: n_q * 32].contiguous(), [32] * n_q
        for name, allow in masks.items():
            a, b, same, stats = measure(idx, q_dev, q_lens, allow)
            nbytes = stats["rows"] * idx.row_bytes
            assert stats["rows"] == int(allow.sum()) * bench.P_PATCH, (stats, int(allow.sum()))
            out["results"].append({"dtype": dt, "queries": n_q, "mask": name, "allowed_pages": int(allow.sum()),
                                   "filtered_ms_p50": round(a, 4), "scan_all_ms_p50": round(b, 4),
                                   "algorithmic_bytes": nbytes, "filtered_call_gb_per_s": round(nbytes / a / 1e6, 1),
                                   "units": stats["units"], "bit_identical": bool(same)})
    idx.close()
print(json.dumps(out))
