"""Small driver for ncu captures (NOT a benchmark: numbers printed under a profiler are never bench values).

Builds a synthetic shard (default 32768 pages x 1024 x 128, 8.6 GB bf16) and launches each scoring kernel a few times
in a fixed order so that `ncu -k regex:<name> -s <skip> -c <count>` picks a warm launch:
  (default)     bf16: 4x bq=32 (maxsim_wgmma<0,4>), then 4x bq=1 (maxsim_wgmma<0,1>)
  --only int8   int8 sub-shard: 4x bq=32 (maxsim_wgmma<1,4>), 4x bq=1
  --only fp8    fp8 sub-shard, same
  --only binary 1-bit sub-shard: 4x bq=8 (wgmma path), 4x bq=1 (POPC path)
  --only fde    FDE matrix of the shard: 4x scan with 1 query, 4x with 32 queries (fde_scan_wgmma_kernel)
"""
import argparse
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

import torch  # noqa: E402

import bench  # noqa: E402
from morphik_core_b200.index import MaxSimIndex  # noqa: E402

ap = argparse.ArgumentParser()
ap.add_argument("--pages", type=int, default=32768)
ap.add_argument("--only", choices=["bf16", "int8", "fp8", "binary", "fde"], default="bf16")
ap.add_argument("--reps", type=int, default=4)
ap.add_argument("--bqs", type=str, default="32,1", help="query batch sizes to drive")
args = ap.parse_args()

dev = torch.device("cuda", 0)
q_host = bench.make_queries(32)
packed, _ = bench.build_shard(args.pages, dev, 1234, q_host)
q_dev = q_host.to(dev)
lens = [bench.P_PATCH] * args.pages


def drive(idx, bqs):
    for bq in bqs:
        q = q_dev[: bq * 32].contiguous()
        for _ in range(args.reps):
            idx.search_device(q, [32] * bq, 10)
        torch.cuda.synchronize()
        ms = idx.score_times_ms(args.reps)
        print(f"{idx.dtype_name} bq={bq}: score ms {['%.3f' % m for m in ms]}", flush=True)


if args.only == "bf16":
    idx = MaxSimIndex(dtype="bf16")
    idx.adopt_packed(packed, lens)
    drive(idx, [int(b) for b in args.bqs.split(",")])
elif args.only in ("int8", "fp8"):
    drive(bench.quantised_subshard(packed, args.pages, args.only, 0), [int(b) for b in args.bqs.split(",")])
elif args.only == "binary":
    drive(bench.quantised_subshard(packed, args.pages, "binary", 0), [int(b) for b in args.bqs.split(",")] if args.bqs != "32,1" else [8, 1])
else:
    from morphik_core_b200.fde import TwoStageIndex

    sub = MaxSimIndex(dtype="bf16")
    sub.adopt_packed(packed, lens)
    two = TwoStageIndex(index=sub)
    two.rebuild_from_index()
    for nq in (1, 32):
        qf = torch.randn((nq, two.fde_dim), device=dev)
        for _ in range(args.reps):
            two.fde_scores(qf)
        torch.cuda.synchronize()
        print(f"fde scan n_q={nq} done", flush=True)
