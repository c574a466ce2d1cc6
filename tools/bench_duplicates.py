"""Near-duplicate detection probe (B200MultiVectorStore.index_duplicates, MaxSimIndex.pair_maxsim / duplicate_groups,
query_similar_distinct) -- NOT the bench.py metric -- on bench.py's topic corpus: 65 536 pages x 1024 patch rows, bf16 and
int8, with planted near-duplicates: copies of 2 % of the pages with row noise at three levels, and copies with 10 % of their
rows dropped.  Both dtypes share one FDE first stage: its rows come from the float pages, so the int8 index takes the bf16
index's FDE rows (as tools/bench_similar.py does).

Per dtype, with the FDE first stage at n_candidates 10 and 20:
  * index_duplicates' wall time split into first stage (TwoStageSearch.duplicate_candidates over every page), pair kernel
    and components (CUDA events around each step);
  * the pair kernel's TFLOP/s: 2 * len_a * len_b * 128 FLOP per pair, counted once (one product serves both directions), over
    its device time from torch.profiler;
  * recall of the planted pairs and the number of other edges at a few thresholds;
  * p50 / p95 of query_similar_distinct against query_similar, alternated, CUDA events around each synchronous call (so
    the device time from the call's first launch to its last, without the event loop), and of the label step alone.
On a slice of --slice sources (bf16): the exhaustive first stage (MaxSimIndex.duplicate_candidates, every source a full
scan), for the cost per source.
Prints the card name and power limit, then one JSON line.

  python tools/bench_duplicates.py [--pages 65536] [--reps 20] [--cands 10,20] [--thresholds 0.8,0.9,0.95] [--slice 128]
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
from morphik_core_b200.fde import TwoStageIndex  # noqa: E402
from morphik_core_b200.index import MaxSimIndex  # noqa: E402
from morphik_core_b200.store import B200MultiVectorStore  # noqa: E402

ap = argparse.ArgumentParser()
ap.add_argument("--pages", type=int, default=65536)
ap.add_argument("--reps", type=int, default=20)
ap.add_argument("--cands", default="10,20")
ap.add_argument("--thresholds", default="0.8,0.9,0.95")
ap.add_argument("--dtypes", default="bf16,int8")
ap.add_argument("--slice", type=int, default=128)
args = ap.parse_args()

if not torch.cuda.is_available():
    sys.exit("bench_duplicates.py needs a CUDA device (H100); nothing is measured without one")
dev = torch.device("cuda", 0)
card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                      capture_output=True, text=True).stdout.strip()
print(f"[bench_duplicates] card: {card}", flush=True)

ROWS = bench.P_PATCH
NOISE = (0.02, 0.05, 0.1)  # row noise of the planted copies, relative to a unit row
anchors = bench.topic_anchors(dev)
q_host, _ = bench.make_topic_queries(8, anchors)
packed, _ = bench.build_shard(args.pages, dev, seed=1234, q_host=q_host, topic_pages=args.pages // 2, anchors=anchors)
queries = [q_host[i * bench.T_TOK:(i + 1) * bench.T_TOK].numpy() for i in range(8)]


def pct(ms):
    return {"p50_ms": round(float(np.median(ms)), 4), "p95_ms": round(float(np.percentile(ms, 95)), 4)}


def event_ms(fn):
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    out = fn()
    b.record()
    b.synchronize()
    return a.elapsed_time(b), out


def kernel_ms(fn, name):
    from torch.profiler import ProfilerActivity, profile

    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    us = sum(getattr(e, "device_time_total", getattr(e, "cuda_time_total", 0)) for e in prof.key_averages() if name in e.key)
    return us / 1e3


def planted_pages(idx, rng):
    """The planted copies as float pages on the device, and the (original, copy) pairs they make once appended."""
    n0 = idx.n_pages
    src = rng.choice(n0, size=max(4, n0 // 50), replace=False)
    pages, pairs = [], []
    for i in range(0, len(src), 64):
        ids = [int(p) for p in src[i:i + 64]]
        rows, lens = idx.page_rows(ids)
        off = 0
        for j, (p, n) in enumerate(zip(ids, lens)):
            x = rows[off:off + n]
            off += n
            kind = (i + j) % 4
            if kind < 3:  # row noise
                x = torch.nn.functional.normalize(x + NOISE[kind] * torch.randn_like(x) / bench.DIM ** 0.5, dim=1)
            else:  # 10 % of the rows dropped
                keep = torch.randperm(n, device=x.device)[: n - n // 10].sort().values
                x = x[keep]
            pages.append(x.contiguous())
            pairs.append((p, n0 + len(pages) - 1))
    return pages, pairs


def add_in_batches(idx, pages):
    for i in range(0, len(pages), 64):
        idx.add_pages(pages[i:i + 64])
    idx._attach()


def run_dtype(dtype, idx, two, planted):
    n = idx.n_pages
    store = B200MultiVectorStore(mode=dtype, index=idx, auto_initialize=False, coalesce_queries=False, fde_candidates=64)
    store._two_stage = two
    for p in range(n):
        store.catalog.add(PageRecord(f"doc{p}", 0, "", {}, None, int(idx.page_lens[p])))
    planted_set = set(planted)
    lens = torch.from_numpy(idx.page_lens.astype(np.int64)).to(dev)
    for n_cand in [int(c) for c in args.cands.split(",")]:
        t_cand, (a, b) = event_ms(lambda: two.duplicate_candidates(list(range(n)), n_cand))
        t_pair, (sab, sba) = event_ms(lambda: idx.pair_maxsim(a, b))
        t_groups, _ = event_ms(lambda: idx.duplicate_groups(a, b, sab, sba, 0.9))
        pk_ms = kernel_ms(lambda: idx.pair_maxsim(a, b), "pair_maxsim")
        flop = float((lens[a] * lens[b]).double().sum().item()) * 2 * bench.DIM
        ah, bh = a.cpu().numpy(), b.cpu().numpy()
        dup = torch.minimum(sab, sba).cpu().numpy()
        found = set(zip(ah.tolist(), bh.tolist())) & planted_set
        per_t = {}
        for t in [float(x) for x in args.thresholds.split(",")]:
            edge = dup >= t
            hit = sum(1 for x, y, e in zip(ah.tolist(), bh.tolist(), edge.tolist()) if e and (x, y) in planted_set)
            per_t[str(t)] = {"planted_recall": round(hit / len(planted), 4), "other_edges": int(edge.sum()) - hit}
        row = {"dtype": dtype, "n_candidates": n_cand, "pairs": int(a.numel()), "first_stage_ms": round(t_cand, 1),
               "pair_kernel_call_ms": round(t_pair, 1), "components_ms": round(t_groups, 3),
               "pair_kernel_device_ms": round(pk_ms, 1),
               "pair_tflops": round(flop / (pk_ms * 1e-3) / 1e12, 1) if pk_ms > 0 else None,
               "planted_pairs": len(planted), "planted_in_candidates": len(found), "thresholds": per_t}
        print(f"[bench_duplicates] {json.dumps(row)}", flush=True)
        results.append(row)
        del a, b, sab, sba
    # the table of the last n_candidates, through the store; then the per-request search
    asyncio.run(store.index_duplicates(n_candidates=int(args.cands.split(",")[-1]), rebuild=True))
    t = 0.9
    d = store._dup
    label_ms = [event_ms(lambda: idx.duplicate_groups(d["a"], d["b"], d["sab"], d["sba"], t))[0] for _ in range(args.reps)]
    distinct, flat = [], []
    for i in range(3 + args.reps):
        q = queries[i % len(queries)]
        t_d, _ = event_ms(lambda: asyncio.run(store.query_similar_distinct(q, k=10, threshold=t)))
        t_f, _ = event_ms(lambda: asyncio.run(store.query_similar(q, k=10)))
        if i >= 3:
            distinct.append(t_d)
            flat.append(t_f)
    row = {"dtype": dtype, "table_pairs": int(d["a"].numel()), "threshold": t, "label_step": pct(label_ms),
           "query_similar_distinct": pct(distinct), "query_similar": pct(flat)}
    print(f"[bench_duplicates] {json.dumps(row)}", flush=True)
    results.append(row)
    store._dup = None


results = []
rng = np.random.default_rng(7)
fde_bf16 = TwoStageIndex(dtype="bf16")
fde_bf16.adopt_packed(packed, [ROWS] * args.pages)
idx16 = fde_bf16.index
idx16._attach()
extra, planted = planted_pages(idx16, rng)
for i in range(0, len(extra), 64):
    fde_bf16.add_pages(extra[i:i + 64])
idx16._attach()
for dtype in args.dtypes.split(","):
    if dtype == "bf16":
        idx, two = idx16, fde_bf16
    else:
        idx = bench.quantised_subshard(packed, args.pages, dtype, 0)
        add_in_batches(idx, extra)
        two = TwoStageIndex(index=idx)  # the same FDE rows: they come from the float pages, not the corpus dtype
        two.append_fde_rows(*fde_bf16.fde_rows())
    run_dtype(dtype, idx, two, planted)
    if dtype != "bf16":
        del idx, two
        torch.cuda.empty_cache()

# the exhaustive first stage on a slice of sources: every source's rows are one full scan of the corpus
src = list(range(args.slice))
t_ex, (a, b) = event_ms(lambda: idx16.duplicate_candidates(src, 10))
row = {"dtype": "bf16", "slice_sources": len(src), "mode": "exhaustive", "n_candidates": 10, "pairs": int(a.numel()),
       "first_stage_ms": round(t_ex, 1), "ms_per_source": round(t_ex / len(src), 2)}
print(f"[bench_duplicates] {json.dumps(row)}", flush=True)
results.append(row)

print(json.dumps({"workload": f"{args.pages} pages x {ROWS} patches + 2 % planted copies, FDE first stage, k 10",
                  "card": card, "results": results}))
