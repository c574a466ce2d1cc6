"""Check every page of bench.py's own shard against the float64 MaxSim reference (one H100; not part of the test suite).

Rebuilds the resident bf16 shard with bench.build_shard exactly as bench.py does (163 840 pages x 1024 rows by default,
42.9 GB, topic pages, planted pages), scores 32 queries on it with MaxSimIndex.score_matrix and compares every page with
tests/scale_reference.reference_scores (computed on the GPU from the packed bytes the scan reads), and the top-10 of
search_host with the reference ranking.  Prints one JSON line: pages checked, the largest error against the bf16 tolerance of
oracle.scoring and pass / fail.

    python tools/check_bench_shard.py [--pages N] [--queries 32]
"""
import argparse
import json
import os
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "tests")]

import numpy as np  # noqa: E402
import torch  # noqa: E402

import bench  # noqa: E402
import scale_reference as sr  # noqa: E402
from morphik_core_b200.index import MaxSimIndex  # noqa: E402
from oracle.scoring import TOL, assert_ranking, score_error  # noqa: E402


def main():
    ap = argparse.ArgumentParser(description=__doc__.splitlines()[0])
    ap.add_argument("--pages", type=int, default=163840)
    ap.add_argument("--queries", type=int, default=32)
    ap.add_argument("--k", type=int, default=10)
    args = ap.parse_args()
    device = torch.device("cuda", 0)
    free, total = torch.cuda.mem_get_info(device)
    t0 = time.time()
    q_host = bench.make_queries(args.queries)
    anchors = bench.topic_anchors(device)
    topic_pages = min(65536, args.pages // 2)  # bench.py's --topic-pages default, capped as bench.py caps it
    packed, _ = bench.build_shard(args.pages, device, seed=1234, q_host=q_host, topic_pages=topic_pages, anchors=anchors)
    idx = MaxSimIndex(dtype="bf16")
    idx.adopt_packed(packed, [bench.P_PATCH] * args.pages)
    queries = [q_host[i * bench.T_TOK:(i + 1) * bench.T_TOK].numpy() for i in range(args.queries)]
    lens = [bench.T_TOK] * args.queries
    t1 = time.time()
    got = idx.score_matrix(queries)
    _, goff, _, q_packed = idx.score_groups(queries)
    want = sr.reference_scores(idx, q_packed, goff, lens)
    t2 = time.time()
    err = score_error("bf16", got, want)
    ts, ti, tc = idx.search_host(queries, args.k)
    topk_ok = 0
    for qi in range(args.queries):
        try:
            assert_ranking("bf16", ts[qi], ti[qi], tc[qi], want[qi], args.k)
            topk_ok += 1
        except AssertionError:
            pass
    ok = err <= TOL["bf16"] and topk_ok == args.queries
    print(json.dumps({
        "gpu": torch.cuda.get_device_name(device), "free_gib_at_start": round(free / 2**30, 1),
        "pages_checked": int(got.shape[1]), "queries": args.queries, "shard_gb": round(idx.n_rows_padded * 256 / 1e9, 1),
        "max_rel_err": err, "tolerance": TOL["bf16"], "topk_lists_matching": f"{topk_ok}/{args.queries}",
        "build_s": round(t1 - t0, 1), "score_and_reference_s": round(t2 - t1, 1), "pass": bool(ok)}))
    return 0 if ok else 1


if __name__ == "__main__":
    sys.exit(main())
