"""B200MultiVectorStore.query_similar_mmr without a GPU: argument rules and the routing of the fetch, the masks and the
MMR call through an injected index (exhaustive) and an injected first stage (two-stage), in the pattern of
test_sign_store_cpu.py (test wiring only; the product builds the CUDA index)."""
import asyncio

import numpy as np
import pytest
import torch

from morphik_core_b200.models import DocumentChunk
from morphik_core_b200.store import B200MultiVectorStore


def _allowed(n, allow_mask):
    if allow_mask is None:
        return list(range(n))
    bits = np.unpackbits(np.asarray(allow_mask, np.uint32).view(np.uint8), bitorder="little")
    return [p for p in range(n) if bits[p]]


class FakeIndex:
    """Answers a search with every allowed page, best id first, and an MMR call with the candidates in reverse."""
    row_bytes = 256
    device = "cpu"

    def __init__(self):
        self.n = 0
        self.calls = []

    def add_pages(self, pages):
        first = self.n
        self.n += len(pages)
        return first, len(pages)

    def search_host(self, queries, k, allow_mask=None):
        self.calls.append(("search", len(queries), k, None if allow_mask is None else allow_mask.tolist()))
        ids = _allowed(self.n, allow_mask)[:k]
        ts = np.full((len(queries), k), -np.inf, np.float32)
        ti = np.full((len(queries), k), -1, np.int64)
        ts[:, :len(ids)] = np.arange(len(ids), 0, -1)
        ti[:, :len(ids)] = ids
        return ts, ti, np.full(len(queries), len(ids), np.int32)

    def mmr(self, cand_ids, cand_scores, q_lens, k, lambda_mult, with_sims=False):
        assert isinstance(cand_ids, torch.Tensor) and cand_ids.dtype == torch.int64 and cand_scores.dtype == torch.float32
        self.calls.append(("mmr", cand_ids.tolist(), cand_scores.tolist(), list(q_lens), k, lambda_mult))
        n = cand_ids.shape[1]
        order = list(range(n - 1, -1, -1))[:k]
        return cand_ids[:, order], cand_scores[:, order], torch.tensor([len(order)], dtype=torch.int32)


class FakeStage:
    def __init__(self, index):
        self.index = index
        self.calls = []
        self.last_timing_ms = {}

    def add_pages(self, pages):
        return self.index.add_pages(pages)

    def search(self, queries, k, n_candidates=1000, allow_mask=None):
        self.calls.append(("search", k, n_candidates, None if allow_mask is None else allow_mask.tolist()))
        self.last_timing_ms = {"sign_candidates_ms": 1.0}
        return self.index.search_host(queries, k, allow_mask)


def run(coro):
    return asyncio.run(coro)


def _store(two_stage=False, n=9):
    idx = FakeIndex()
    kw = {"sign_candidates": 50} if two_stage else {}
    store = B200MultiVectorStore(auto_initialize=False, index=idx, coalesce_queries=False, **kw)
    if two_stage:
        store._two_stage = FakeStage(idx)
    emb = np.ones((3, 128), np.float32)
    if n:
        run(store.store_embeddings([DocumentChunk(document_id=f"d{i % 3}", chunk_number=i, content=str(i), embedding=emb,
                                                  metadata={}) for i in range(n)]))
    return store, idx


Q = np.ones((5, 128), np.float32)


@pytest.mark.parametrize("two_stage", [False, True])
def test_fetch_then_mmr_with_masks(two_stage):
    store, idx = _store(two_stage)
    res = run(store.query_similar_mmr(Q, k=3, fetch_k=6, lambda_mult=0.25))
    # the fake MMR reverses the 6 fetched candidates: pages 5, 4, 3 with their search scores 1, 2, 3
    assert [(r.chunk_number, r.score) for r in res] == [(5, 1.0), (4, 2.0), (3, 3.0)]
    search = [c for c in idx.calls if c[0] == "search"][-1]
    assert search[2] == 6 and search[3] is None
    mmr = idx.calls[-1]
    assert mmr[0] == "mmr" and mmr[1] == [[0, 1, 2, 3, 4, 5]] and mmr[3] == [5] and mmr[4] == 3 and mmr[5] == 0.25
    if two_stage:
        assert store._two_stage.calls[-1][:3] == ("search", 6, 50)
        assert store.last_query_timing["sign_candidates_ms"] == 1.0
    assert "mmr_ms" in store.last_query_timing
    # doc_ids: the mask reaches the fetch, and only its pages reach the MMR
    res = run(store.query_similar_mmr(Q, k=2, fetch_k=20, doc_ids=["d1"]))  # d1 = pages 1, 4, 7
    search = [c for c in idx.calls if c[0] == "search"][-1]
    assert search[3] == [0b10010010]
    assert idx.calls[-1][1] == [[1, 4, 7]] and idx.calls[-1][4] == 2
    assert {r.document_id for r in res} == {"d1"}
    assert run(store.query_similar_mmr(Q, k=2, doc_ids=["nope"])) == []


def test_fetch_k_below_k_fetches_k():
    store, idx = _store()
    res = run(store.query_similar_mmr(Q, k=4, fetch_k=2))
    assert len(res) == 4
    assert [c for c in idx.calls if c[0] == "search"][-1][2] == 4
    # k past the corpus: everything, once
    res = run(store.query_similar_mmr(Q, k=50, fetch_k=100))
    assert sorted(r.chunk_number for r in res) == list(range(9))
    assert [c for c in idx.calls if c[0] == "search"][-1][2] == 9


def test_empty_store_and_k_zero():
    store, idx = _store(n=0)
    assert run(store.query_similar_mmr(Q, k=3)) == []
    store, idx = _store()
    assert run(store.query_similar_mmr(Q, k=0)) == []
    assert not [c for c in idx.calls if c[0] == "mmr"]


@pytest.mark.parametrize("lam", [-0.01, 1.01, float("nan"), float("inf")])
def test_lambda_outside_unit_interval_is_refused(lam):
    store, idx = _store()
    with pytest.raises(ValueError, match="lambda_mult"):
        run(store.query_similar_mmr(Q, k=3, lambda_mult=lam))
    assert not [c for c in idx.calls if c[0] in ("mmr", "search")]


def test_lambda_bounds_are_accepted():
    store, idx = _store()
    for lam in (0.0, 1.0):
        assert len(run(store.query_similar_mmr(Q, k=2, lambda_mult=lam))) == 2
        assert idx.calls[-1][5] == lam


def test_sharded_store_has_no_mmr():
    from morphik_core_b200.sharded_store import ShardedB200MultiVectorStore

    assert not hasattr(ShardedB200MultiVectorStore, "query_similar_mmr")
