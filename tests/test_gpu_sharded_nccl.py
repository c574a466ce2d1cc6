"""2-GPU (NCCL) test of the document-sharded search: every rank scans only its shard on its own GPU, one all-gather of
the per-shard top-k, merge on the device -- and every rank must end up with the oracle's global top-k.
Skipped on boxes with fewer than 2 GPUs (the host logic is covered on CPU by tests/test_sharded_gloo.py)."""
import os
import socket

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

torch = pytest.importorskip("torch")
if not torch.cuda.is_available():  # pragma: no cover
    pytest.skip("CUDA device required", allow_module_level=True)

import torch.distributed as dist  # noqa: E402
import torch.multiprocessing as mp  # noqa: E402


def _free_port():
    with socket.socket() as s:
        s.bind(("127.0.0.1", 0))
        return s.getsockname()[1]


def _watchdog(seconds=90):
    import faulthandler
    import sys

    faulthandler.dump_traceback_later(seconds, exit=True, file=sys.stderr)  # a hung collective must not burn the GPU lease


def _worker(rank, world, port, mode, result_dir):
    _watchdog()
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    torch.cuda.set_device(rank)
    dist.init_process_group("nccl", rank=rank, world_size=world, device_id=torch.device("cuda", rank))
    try:
        from morphik_core_b200.index import MaxSimIndex
        from morphik_core_b200.sharded import ShardedMaxSim, plan_document_shards
        from oracle import maxsim_oracle as orc

        rng = np.random.default_rng(2024)  # identical corpus description on every rank
        doc_pages = rng.integers(1, 8, size=60).tolist()
        page_lens = [int(x) for x in rng.integers(1, 300, size=sum(doc_pages))]
        pages = []
        for n in page_lens:
            x = rng.standard_normal((n, 128)).astype(np.float32)
            pages.append(x / np.linalg.norm(x, axis=1, keepdims=True))
        queries = []
        for t in (32, 32, 12, 40):
            x = rng.standard_normal((t, 128)).astype(np.float32)
            queries.append(x / np.linalg.norm(x, axis=1, keepdims=True))
        first = np.concatenate([[0], np.cumsum(doc_pages)])
        doc_rows = [sum(page_lens[first[d]:first[d + 1]]) for d in range(len(doc_pages))]
        plan = plan_document_shards(doc_rows, world)
        p0, p1 = int(first[plan[rank][0]]), int(first[plan[rank][1]])

        idx = MaxSimIndex(device=rank, dtype=mode)
        idx.add_pages(pages[p0:p1])
        sharded = ShardedMaxSim.from_index(idx, id_base=p0)
        q = torch.from_numpy(np.concatenate(queries)).cuda()
        if rank != 0:
            q.zero_()
        q = sharded.broadcast_queries(q, src=0)
        k = 9
        ts, ti, tc = sharded.search(q, [len(x) for x in queries], k)
        torch.cuda.synchronize()
        ts, ti = ts.cpu().numpy(), ti.cpu().numpy()
        rows = np.concatenate(pages)
        off = orc.page_offsets(page_lens)
        for qi, qq in enumerate(queries):
            if mode == "bf16":
                want = orc.float_maxsim_c(orc.bf16_round_np(qq), orc.bf16_round_np(rows), off)
            else:
                want = orc.binary_maxsim_c(orc.sign_pack_c(qq), orc.sign_pack_c(rows), off)[0]
            ws, wi = orc.topk_np(want, k)
            assert ti[qi].tolist() == wi.tolist(), (rank, qi, ti[qi].tolist(), wi.tolist())
            np.testing.assert_allclose(ts[qi], ws, rtol=3e-5)
        # pipelined form: three steps, two tickets in flight, each step's result picked up one step later
        outs, tickets = [], []
        for step in range(3):
            t, out = sharded.begin(q, [len(x) for x in queries], k)
            tickets.append(t)
            outs.append(out)
            if step:
                sharded.end(tickets[step - 1])
        sharded.end(tickets[-1])
        torch.cuda.synchronize()
        for o in outs:
            assert np.array_equal(o[1].cpu().numpy(), ti) and np.array_equal(o[0].cpu().numpy(), ts)
        # every rank holds the identical merged list (all-reduce of a checksum)
        chk = torch.stack([outs[-1][1].sum(), outs[-1][1].sum()]).double()
        lo, hi = chk.clone(), chk.clone()
        dist.all_reduce(lo, op=dist.ReduceOp.MIN); dist.all_reduce(hi, op=dist.ReduceOp.MAX)
        assert torch.equal(lo, hi)
        open(os.path.join(result_dir, f"ok{rank}"), "w").write("ok")
    finally:
        dist.destroy_process_group()


@pytest.mark.parametrize("mode", ["bf16", "binary"])
def test_sharded_search_world2_nccl(tmp_path, mode):
    if torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    mp.spawn(_worker, args=(2, _free_port(), mode, str(tmp_path)), nprocs=2, join=True)
    assert sorted(os.listdir(tmp_path)) == ["ok0", "ok1"]


def _store_worker(rank, world, port, result_dir):
    import asyncio

    _watchdog()
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    torch.cuda.set_device(rank)
    dist.init_process_group("nccl", rank=rank, world_size=world, device_id=torch.device("cuda", rank))
    try:
        from morphik_core_b200.models import DocumentChunk
        from morphik_core_b200.sharded_store import ShardedB200MultiVectorStore
        from oracle import maxsim_oracle as orc

        store = ShardedB200MultiVectorStore(mode="bf16")
        if rank != 0:
            store.worker_loop()
            open(os.path.join(result_dir, f"ok{rank}"), "w").write("ok")
            return
        run = asyncio.run
        rng = np.random.default_rng(31)
        docs = {}
        for d in range(16):
            pages = []
            for _ in range(int(rng.integers(1, 6))):
                x = rng.standard_normal((int(rng.integers(5, 300)), 128)).astype(np.float32)
                pages.append(x / np.linalg.norm(x, axis=1, keepdims=True))
            docs[f"doc{d}"] = pages
            run(store.store_embeddings([DocumentChunk(document_id=f"doc{d}", content=f"{d}/{j}", embedding=p, chunk_number=j)
                                        for j, p in enumerate(pages)]))
        assert set(store.doc_rank.values()) == {0, 1}

        def oracle(q, k, allowed=None):
            flat = [(d, j, p) for d, ps in docs.items() for j, p in enumerate(ps) if allowed is None or d in allowed]
            rows = orc.bf16_round_np(np.concatenate([p for _, _, p in flat]))
            s = orc.float_maxsim_c(orc.bf16_round_np(q), rows, orc.page_offsets([len(p) for _, _, p in flat]))
            order = np.argsort(-s.astype(np.float64), kind="stable")[:k]
            return [(flat[i][0], flat[i][1]) for i in order], s[order]

        q = rng.standard_normal((32, 128)).astype(np.float32)
        res = run(store.query_similar(q, k=10))
        want, ws = oracle(q, 10)
        assert [(r.document_id, r.chunk_number) for r in res] == want
        np.testing.assert_allclose([r.score for r in res], ws, rtol=3e-5)
        on1 = [d for d, r in store.doc_rank.items() if r == 1][:3]
        res = run(store.query_similar(q, k=50, doc_ids=on1))
        assert [(r.document_id, r.chunk_number) for r in res] == oracle(q, 50, set(on1))[0]
        # concurrent callers, different filters: one coalesced command, per-query masks on every GPU
        on0 = [d for d, r in store.doc_rank.items() if r == 0][:2]
        reqs = [dict(query_embedding=q, k=10), dict(query_embedding=q, k=50, doc_ids=on1), dict(query_embedding=q, k=4, doc_ids=on0),
                dict(query_embedding=docs["doc3"][0][:20], k=5, doc_ids=on0 + on1), dict(query_embedding=q, k=3, doc_ids=["nope"])]

        async def many():
            return await asyncio.gather(*[store.query_similar(**r) for r in reqs])

        together = run(many())
        assert store.last_coalesced_batch == len(reqs) and together[4] == []
        assert [(r.document_id, r.chunk_number) for r in together[0]] == want
        assert [(r.document_id, r.chunk_number) for r in together[1]] == oracle(q, 50, set(on1))[0]
        assert [(r.document_id, r.chunk_number) for r in together[2]] == oracle(q, 4, set(on0))[0]
        assert [(r.document_id, r.chunk_number) for r in together[3]] == oracle(docs["doc3"][0][:20], 5, set(on0 + on1))[0]
        for d in list(docs)[:7]:
            run(store.delete_chunks_by_document_id(d))
            docs.pop(d)
        res = run(store.query_similar(q, k=10))
        assert [(r.document_id, r.chunk_number) for r in res] == oracle(q, 10)[0]
        store.close()
        open(os.path.join(result_dir, "ok0"), "w").write("ok")
    finally:
        dist.destroy_process_group()


def _two_stage_store_worker(rank, world, port, result_dir):
    import asyncio

    _watchdog()
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    torch.cuda.set_device(rank)
    dist.init_process_group("nccl", rank=rank, world_size=world, device_id=torch.device("cuda", rank))
    try:
        from morphik_core_b200.models import DocumentChunk
        from morphik_core_b200.sharded_store import ShardedB200MultiVectorStore
        from oracle import maxsim_oracle as orc

        # fde_candidates larger than any shard: the two-stage path degenerates to the exhaustive answer (checkable)
        store = ShardedB200MultiVectorStore(mode="bf16", fde_candidates=500)
        if rank != 0:
            store.worker_loop()
            open(os.path.join(result_dir, f"ok{rank}"), "w").write("ok")
            return
        run = asyncio.run
        rng = np.random.default_rng(37)
        docs = {}
        for d in range(40):
            pages = []
            for _ in range(int(rng.integers(2, 6))):
                x = rng.standard_normal((int(rng.integers(32, 200)), 128)).astype(np.float32)
                pages.append(x / np.linalg.norm(x, axis=1, keepdims=True))
            docs[f"doc{d}"] = pages
            run(store.store_embeddings([DocumentChunk(document_id=f"doc{d}", content=f"{d}/{j}", embedding=p, chunk_number=j)
                                        for j, p in enumerate(pages)]))
        flat = [(d, j, p) for d, ps in docs.items() for j, p in enumerate(ps)]
        rows = orc.bf16_round_np(np.concatenate([p for _, _, p in flat]))
        off = orc.page_offsets([len(p) for _, _, p in flat])
        for t in (32, 20):
            q = rng.standard_normal((t, 128)).astype(np.float32)
            s = orc.float_maxsim_c(orc.bf16_round_np(q), rows, off)
            order = np.argsort(-s.astype(np.float64), kind="stable")[:7]
            res = run(store.query_similar(q, k=7))
            assert [(r.document_id, r.chunk_number) for r in res] == [(flat[i][0], flat[i][1]) for i in order]
            np.testing.assert_allclose([r.score for r in res], s[order], rtol=3e-5)
        assert {"encode_query_ms", "ns_query_ms", "rerank_scoring_ms", "total_ms"} <= set(store.last_query_timing)
        on1 = [d for d, r in store.doc_rank.items() if r == 1][:5]
        res = run(store.query_similar(q, k=30, doc_ids=on1))
        assert {r.document_id for r in res} <= set(on1) and len(res) == min(30, sum(len(docs[d]) for d in on1))
        store.close()
        open(os.path.join(result_dir, "ok0"), "w").write("ok")
    finally:
        dist.destroy_process_group()


def test_sharded_two_stage_store_world2_nccl(tmp_path):
    if torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    mp.spawn(_two_stage_store_worker, args=(2, _free_port(), str(tmp_path)), nprocs=2, join=True)
    assert sorted(os.listdir(tmp_path)) == ["ok0", "ok1"]


def test_sharded_store_world2_nccl(tmp_path):
    if torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    mp.spawn(_store_worker, args=(2, _free_port(), str(tmp_path)), nprocs=2, join=True)
    assert sorted(os.listdir(tmp_path)) == ["ok0", "ok1"]
