"""Asymmetric sign candidates vs the FDE scan vs symmetric Hamming as the first stage of a two-stage search, on one GPU.
Prints one JSON line.

  python tools/bench_sign_stage.py [--pages 65536] [--iters 30] [--recall-queries 32] [--host-pages 65536]

Corpus: bench.build_shard's topic model over every page (65 536 pages x 1024 rows bf16 = 17.2 GB), queries from
bench.make_topic_queries (32 tokens each), so "recall of the exhaustive top-10 among the candidates" is a graded number.
  * latency: p50 / p95 of each first stage alone (CUDA events) and of the whole two-stage search (host clock around a
    synchronised call), 1 and 32 queries, 1000 candidates; the stages are alternated query by query;
  * recall@10 of the exhaustive bf16 MaxSim top-10 with 10, 20, 75 and 1000 candidates for asymmetric signs (at three query scales),
    FDE (TwoStageIndex) and symmetric Hamming (a 1-bit MaxSimIndex over the same sign rows, its own full-scan search);
  * the same signs in front of a host-resident copy of the corpus: latency with the PCIe gather split out (gather_stats) and
    identity of the results with the HBM tier.
Clocks and power: nvidia-smi samples during the timed loops (bench.ClockSampler) and the card's name and power limit.
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
from morphik_core_b200.index import MaxSimIndex  # noqa: E402
from morphik_core_b200.signs import SignTwoStageIndex  # noqa: E402

ap = argparse.ArgumentParser()
ap.add_argument("--pages", type=int, default=65536)
ap.add_argument("--host-pages", type=int, default=65536, help="pages of the host-tier copy (0: skip the host tier)")
ap.add_argument("--iters", type=int, default=30)
ap.add_argument("--recall-queries", type=int, default=32)
ap.add_argument("--k", type=int, default=10)
ap.add_argument("--scales", default="32,127,512")
args = ap.parse_args()

dev = torch.device("cuda", 0)
T = bench.T_TOK
k = args.k
anchors = bench.topic_anchors(dev)
n_lat = max(64, args.iters)
tq_host, _ = bench.make_topic_queries(n_lat + args.recall_queries, anchors)
queries = [tq_host[i * T:(i + 1) * T] for i in range(n_lat + args.recall_queries)]
lat_q, rec_q = queries[:n_lat], queries[n_lat:]
packed, _ = bench.build_shard(args.pages, dev, 1234, bench.make_queries(1), planted_per_query=0, topic_pages=args.pages,
                              anchors=anchors)
lens = [bench.P_PATCH] * args.pages
idx = MaxSimIndex(dtype="bf16")
idx.adopt_packed(packed, lens)
t0 = time.perf_counter()
sig = SignTwoStageIndex(index=idx)
sig.rebuild_from_index()
torch.cuda.synchronize()
sign_build_s = time.perf_counter() - t0
t0 = time.perf_counter()
fde = TwoStageIndex(index=idx)
fde.rebuild_from_index()
torch.cuda.synchronize()
fde_build_s = time.perf_counter() - t0
ham = MaxSimIndex(dtype="binary")  # symmetric Hamming MaxSim over the very same sign rows
ham.adopt_packed(sig.sign_rows(), lens)
scale_default = sig.q_scale


def dev_q(qs):
    return torch.cat(qs).to(dev).contiguous(), [T] * len(qs)


def ham_candidates(qs, n_cand):
    src, ql = dev_q(qs)
    return ham.search_device(src, ql, n_cand)[1]


# ---- recall@k of the exhaustive top-k among each first stage's candidates (the rerank keeps exactly those pages)
src_r, lens_r = dev_q(rec_q)
truth = idx.search_device(src_r, lens_r, k)[1].cpu().numpy()


def recall(cand_ids):
    c = cand_ids.cpu().numpy()
    return float(np.mean([len(set(truth[q].tolist()) & set(c[q].tolist())) / k for q in range(len(rec_q))]))


rec = {}
for n_cand in (10, 20, 75, 1000):  # 10 and 20 as well: the topic corpus saturates every first stage at 75
    for s in [float(x) for x in args.scales.split(",")]:
        sig.q_scale = s
        rec[f"signs_q{s:g}_c{n_cand}"] = recall(sig.candidates_device(src_r, lens_r, n_cand)[1])
    sig.q_scale = scale_default
    rec[f"fde_c{n_cand}"] = recall(fde.candidates(rec_q, n_cand)[0])
    rec[f"hamming_c{n_cand}"] = recall(ham_candidates(rec_q, n_cand))
    # end to end: the two-stage top-k against the exhaustive top-k
    rec[f"signs_two_stage_c{n_cand}"] = recall(sig.search_device(rec_q, k, n_cand)[1])
    rec[f"fde_two_stage_c{n_cand}"] = recall(fde.search_device(rec_q, k, n_cand)[1])


# ---- latency, stages alternated query by query
def pct(v):
    v = np.sort(np.asarray(v))
    return {"p50": float(v[len(v) // 2]), "p95": float(v[min(len(v) - 1, int(len(v) * 0.95))]),
            "min": float(v[0]), "max": float(v[-1])}


def stage_ms(fn):
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    fn()
    e1.record()
    e1.synchronize()
    return e0.elapsed_time(e1)


def wall_ms(fn):
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    fn()
    torch.cuda.synchronize()
    return (time.perf_counter() - t0) * 1e3


lat = {}
sampler = bench.ClockSampler(0)
sampler.start()
t_lat0 = time.perf_counter()
for n_q in (1, 32):
    groups = [lat_q[i * n_q % n_lat:][:n_q] for i in range(args.iters)]
    dq = [dev_q(g) for g in groups]
    for g, (src, ql) in zip(groups[:3], dq[:3]):  # warm-up of every shape
        sig.candidates_device(src, ql, 1000), fde.candidates(g, 1000), ham.search_device(src, ql, 1000)
        sig.search(g, k, 1000), fde.search(g, k, 1000)
    r = {key: [] for key in ("signs_stage", "fde_stage", "hamming_stage", "signs_two_stage", "fde_two_stage",
                             "signs_two_stage_sign_ms", "signs_two_stage_rerank_ms")}
    for g, (src, ql) in zip(groups, dq):
        r["signs_stage"].append(stage_ms(lambda: sig.candidates_device(src, ql, 1000)))
        r["fde_stage"].append(stage_ms(lambda: fde.candidates(g, 1000)))  # includes the query FDE encode
        r["hamming_stage"].append(stage_ms(lambda: ham.search_device(src, ql, 1000)))
        r["signs_two_stage"].append(wall_ms(lambda: sig.search(g, k, 1000)))
        r["signs_two_stage_sign_ms"].append(sig.last_timing_ms["sign_candidates_ms"])
        r["signs_two_stage_rerank_ms"].append(sig.last_timing_ms["maxsim_rerank_ms"])
        r["fde_two_stage"].append(wall_ms(lambda: fde.search(g, k, 1000)))
    lat[f"q{n_q}_c1000"] = {key: pct(v) for key, v in r.items()}
clocks = sampler.stop(t_lat0, time.perf_counter())

# ---- host tier: the same signs (derived through the mapping) in front of a host-resident copy
host = {}
if args.host_pages:
    hp = min(args.host_pages, args.pages)
    hidx = MaxSimIndex(dtype="bf16", tier="host")
    hidx.adopt_packed(packed[: hp * bench.P_PATCH * 256], lens[:hp])
    t0 = time.perf_counter()
    hsig = SignTwoStageIndex(index=hidx)
    hsig.rebuild_from_index()
    torch.cuda.synchronize()
    host["sign_build_s"] = time.perf_counter() - t0
    host["signs_equal_hbm"] = bool(hp == args.pages and torch.equal(hsig.sign_rows(), sig.sign_rows()))
    identical = True
    for n_q, n_cand in ((1, 75), (1, 1000), (32, 1000)):
        r = {"two_stage": [], "sign_candidates_ms": [], "gather_ms": [], "rerank_scoring_ms": [], "gather_bytes": []}
        for it in range(args.iters):
            g = lat_q[it * n_q % n_lat:][:n_q]
            r["two_stage"].append(wall_ms(lambda: hsig.search(g, k, n_cand)))
            st = hsig.last_timing_ms
            r["sign_candidates_ms"].append(st["sign_candidates_ms"])
            r["gather_ms"].append(st["load_multivectors_ms"])
            r["rerank_scoring_ms"].append(st["rerank_scoring_ms"])
            r["gather_bytes"].append(st["gather_bytes"])
            if it < 3 and hp == args.pages:
                a, b = hsig.search(g, k, n_cand), sig.search(g, k, n_cand)
                identical &= all(np.array_equal(x.view(np.int32) if x.dtype == np.float32 else x, y.view(np.int32) if
                                                y.dtype == np.float32 else y) for x, y in zip(a, b))
        host[f"q{n_q}_c{n_cand}"] = {key: pct(v[3:]) for key, v in r.items()}
    host["identical_to_hbm_tier"] = identical
    host["pages"] = hp
    hidx.close()

print(json.dumps({
    "gpu": bench.gpu_name_and_power_limit(0), "clocks_during_latency": clocks,
    "workload": f"{args.pages} pages x {bench.P_PATCH} rows bf16 ({args.pages * bench.P_PATCH * 256 / 1e9:.1f} GB), sign rows "
                f"{args.pages * bench.P_PATCH * 16 / 1e9:.2f} GB, FDE matrix {args.pages * fde.fde_dim * 2 / 1e9:.2f} GB; topic "
                f"queries of {T} tokens; top-{k}",
    "build_s": {"signs": sign_build_s, "fde": fde_build_s}, "q_scale_default": scale_default,
    "recall_at_k": rec, "recall_queries": len(rec_q), "latency_ms": lat, "host_tier": host,
    "notes": "stage = first stage alone (CUDA events; FDE includes the query encode); two_stage = host clock around "
             "search() incl. staging and the copy of the results; recall = share of the exhaustive bf16 top-k among the "
             "candidates (or in the two-stage top-k)"}))
