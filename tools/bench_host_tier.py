"""Host-resident corpus probe (NOT the bench.py metric): the patch rows of a bf16 shard in pinned host memory, the FDE matrix in
HBM, and per search a PCIe gather of only the candidate pages.  Prints one JSON line:

  h2d_contiguous_gbs   cudaMemcpyAsync of 1 GiB from the host block (CUDA events): the bar for the gather
  gather_gbs           the gather of 1000 distinct random 1024-row pages (unique pages x padded rows x 256 B per ms)
  cases                p50 / p95 end-to-end latency and the stage split of a two-stage search (one 32-token query x 75
                       candidates, the reference's cap; one query x 1000; 32 queries x 1000 each), top-k identical to the
                       same search over an HBM-resident copy of the rows

  python tools/bench_host_tier.py [--pages 65536] [--iters 30]

--pages 65536 pins 17 GB of host memory; the machine's MemAvailable is reported beside the size used.
"""
import argparse
import json
import os
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

import numpy as np  # noqa: E402
import torch  # noqa: E402

import bench  # noqa: E402
from morphik_core_b200.fde import TwoStageIndex  # noqa: E402

ap = argparse.ArgumentParser()
ap.add_argument("--pages", type=int, default=65536)
ap.add_argument("--iters", type=int, default=30)
ap.add_argument("--k", type=int, default=10)
args = ap.parse_args()


def mem_available_gb():
    with open("/proc/meminfo") as f:
        for line in f:
            if line.startswith("MemAvailable:"):
                return int(line.split()[1]) / 1e6
    return None


def pct(xs, p):
    return float(np.percentile(xs, p))


dev = torch.device("cuda", 0)
mem_before = mem_available_gb()
q_host = bench.make_queries(32)
queries = [q_host[i * 32:(i + 1) * 32].numpy() for i in range(32)]
packed, _ = bench.build_shard(args.pages, dev, 1234, q_host, planted_per_query=10)
lens = [bench.P_PATCH] * args.pages
hbm = TwoStageIndex(dtype="bf16")
hbm.adopt_packed(packed, lens)
host = TwoStageIndex(dtype="bf16", tier="host")
host.adopt_packed(packed, lens)  # the rows move into an exactly sized pinned block; the FDE matrix is built on the GPU
torch.cuda.synchronize()
free_hbm, total_hbm = torch.cuda.mem_get_info(dev)

# ---- the bar: contiguous H2D from the same pinned block
blk = host.index._buf
n_h2d = min(1 << 30, blk.numel())
dst = torch.empty(n_h2d, dtype=torch.uint8, device=dev)
h2d = []
for _ in range(6):
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    dst.copy_(blk[:n_h2d], non_blocking=True)
    e1.record()
    e1.synchronize()
    h2d.append(n_h2d / (e0.elapsed_time(e1) * 1e6))
del dst
h2d_gbs = float(np.median(h2d[1:]))

# ---- the gather of 1000 distinct random pages (one query, shared list)
rng = np.random.default_rng(7)
qd = torch.from_numpy(queries[0]).to(dev)
gather = []
for _ in range(args.iters):
    cand = torch.from_numpy(rng.choice(args.pages, size=1000, replace=False).astype(np.int64)).to(dev)
    host.index.rerank(qd, [32], cand, args.k)
    st = host.index.gather_stats()
    assert st["unique_pages"] == 1000 and st["bytes"] == 1000 * bench.P_PATCH * 256, st
    gather.append(st["bytes"] / (st["ms"] * 1e6))
gather_gbs = float(np.median(gather[2:]))


# ---- end-to-end two-stage searches
def dedup_plan_ms(fn):
    """Device time of the dedup / plan kernels of one call (torch.profiler, CUDA activities)."""
    from torch.profiler import ProfilerActivity, profile

    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    names = ("ht_mark", "ht_scan", "ht_compact", "ht_round_plan", "ht_remap")
    return sum(e.device_time_total for e in prof.key_averages() if any(n in e.key for n in names)) / 1e3


cases = {}
identical = True
for name, n_q, n_cand in (("q1_c75", 1, 75), ("q1_c1000", 1, 1000), ("q32_c1000", 32, 1000)):
    qs = queries[:n_q]
    lat, stages = [], []
    for it in range(args.iters):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        s_host, i_host, c_host = host.search(qs, args.k, n_candidates=n_cand)
        lat.append((time.perf_counter() - t0) * 1e3)
        stages.append(dict(host.last_timing_ms))
        if it < 3:
            s_hbm, i_hbm, c_hbm = hbm.search(qs, args.k, n_candidates=n_cand)
            identical &= bool(np.array_equal(i_host, i_hbm) and np.array_equal(s_host.view(np.int32), s_hbm.view(np.int32))
                              and np.array_equal(c_host, c_hbm))
    warm = 3
    lat, stages = lat[warm:], stages[warm:]
    med = lambda key: float(np.median([s[key] for s in stages]))  # noqa: E731
    dp = dedup_plan_ms(lambda: host.search(qs, args.k, n_candidates=n_cand))
    cases[name] = {
        "n_q": n_q, "n_candidates": n_cand, "slots": n_q * n_cand, "unique_pages": int(stages[-1]["gather_pages"]),
        "p50_ms": float(np.median(lat)), "p95_ms": pct(lat, 95),
        "encode_ms": med("encode_query_ms"), "fde_scan_topk_ms": med("ns_query_ms"), "dedup_plan_ms": dp,
        "gather_ms": med("load_multivectors_ms"), "gather_bytes": int(stages[-1]["gather_bytes"]),
        "rerank_ms": med("rerank_scoring_ms") - dp,
    }

gpu = bench.gpu_name_and_power_limit(0)
line = {
    "workload": f"{args.pages} pages x {bench.P_PATCH} patches bf16 in pinned host memory "
                f"({args.pages * bench.P_PATCH * 256 / 1e9:.1f} GB) + FDE matrix in HBM, top-{args.k}",
    "gpu": gpu, "host_tier_gb": args.pages * bench.P_PATCH * 256 / 1e9, "mem_available_gb_before": mem_before,
    "mem_available_gb_after": mem_available_gb(), "hbm_free_gb": free_hbm / 1e9, "hbm_total_gb": total_hbm / 1e9,
    "h2d_contiguous_gbs": h2d_gbs, "gather_gbs": gather_gbs, "gather_vs_h2d": gather_gbs / h2d_gbs,
    "topk_identical_to_hbm": identical, "cases": cases,
}
print(json.dumps(line), flush=True)
