"""B200MultiVectorStore(sign_candidates=N) without a GPU: argument rules and the routing of searches, masks and compaction
through an injected stand-in for signs.SignTwoStageIndex (test wiring only; the product builds the CUDA index)."""
import asyncio

import numpy as np
import pytest

from morphik_core_b200.models import DocumentChunk
from morphik_core_b200.store import B200MultiVectorStore


class FakeIndex:
    row_bytes = 256
    device = "cpu"


class FakeSignStage:
    """Records what the store asks of its first stage and answers with every allowed page, best id first."""

    def __init__(self):
        self.n = 0
        self.calls = []

    def add_pages(self, pages):
        first = self.n
        self.n += len(pages)
        return first, len(pages)

    def compact(self, keep):
        self.calls.append(("compact", list(keep)))
        self.n = len(keep)

    def _allowed(self, allow_mask):
        if allow_mask is None:
            return list(range(self.n))
        bits = np.unpackbits(np.asarray(allow_mask, np.uint32).view(np.uint8), bitorder="little")
        return [p for p in range(self.n) if bits[p]]

    def search(self, queries, k, n_candidates=1000, allow_mask=None):
        self.calls.append(("search", len(queries), k, n_candidates, None if allow_mask is None else allow_mask.tolist()))
        ids = self._allowed(allow_mask)[:k]
        ts = np.full((len(queries), k), -np.inf, np.float32)
        ti = np.full((len(queries), k), -1, np.int64)
        ts[:, :len(ids)] = np.arange(len(ids), 0, -1)
        ti[:, :len(ids)] = ids
        self.last_timing_ms = {"sign_candidates_ms": 1.0, "maxsim_rerank_ms": 2.0, "load_multivectors_ms": 0.5,
                               "rerank_scoring_ms": 1.5}
        return ts, ti, np.full(len(queries), len(ids), np.int32)

    def search_docs(self, queries, k, per_doc, page_doc, n_docs, n_candidates=1000, allow_mask=None):
        self.calls.append(("search_docs", k, per_doc, n_candidates, None if allow_mask is None else allow_mask.tolist()))
        ids = self._allowed(allow_mask)[:k]
        ts = np.full((1, k, per_doc), -np.inf, np.float32)
        ti = np.full((1, k, per_doc), -1, np.int64)
        pc = np.zeros((1, k), np.int32)
        ts[0, :len(ids), 0], ti[0, :len(ids), 0], pc[0, :len(ids)] = 1.0, ids, 1
        return ts, ti, pc, np.array([len(ids)], np.int32)


def run(coro):
    return asyncio.run(coro)


def store_with_fake(n_cand=50, **kw):
    store = B200MultiVectorStore(auto_initialize=False, index=FakeIndex(), sign_candidates=n_cand, coalesce_queries=False, **kw)
    store._two_stage = FakeSignStage()
    return store


def test_first_stages_are_exclusive_and_the_host_tier_takes_either():
    with pytest.raises(ValueError, match="pass one"):
        B200MultiVectorStore(auto_initialize=False, index=FakeIndex(), fde_candidates=10, sign_candidates=10)
    with pytest.raises(ValueError, match="host"):
        B200MultiVectorStore(auto_initialize=False, index=FakeIndex(), corpus_tier="host")
    for kw in ({"sign_candidates": 75}, {"fde_candidates": 75}):
        s = B200MultiVectorStore(auto_initialize=False, index=FakeIndex(), corpus_tier="host", **kw)
        assert s.corpus_tier == "host"
    s = B200MultiVectorStore(auto_initialize=False, index=FakeIndex(), sign_candidates=75)
    assert s.sign_candidates == 75 and not s.fde_candidates


def test_searches_route_through_the_sign_stage_with_masks():
    store = store_with_fake(n_cand=50)
    emb = np.ones((3, 128), np.float32)
    chunks = [DocumentChunk(document_id=f"d{i % 3}", chunk_number=i, content=str(i), embedding=emb, metadata={}) for i in range(9)]
    assert run(store.store_embeddings(chunks))[0]
    st = store._two_stage
    assert st.n == 9
    q = np.ones((2, 128), np.float32)
    res = run(store.query_similar(q, k=4))
    assert [r.chunk_number for r in res] == [0, 1, 2, 3]
    assert st.calls[-1] == ("search", 1, 4, 50, None)
    assert store.last_query_timing["sign_candidates_ms"] == 1.0 and store.last_query_timing["load_multivectors_ms"] == 0.5
    res = run(store.query_similar(q, k=60, doc_ids=["d1"]))  # d1 = pages 1, 4, 7
    assert [r.chunk_number for r in res] == [1, 4, 7]
    _, _, k, n_cand, words = st.calls[-1]
    assert k == 9 and n_cand == 50 and words == [0b10010010]
    res = run(store.query_similar_batch([q, q], k=2, doc_ids=["d2"]))
    assert [[r.chunk_number for r in rr] for rr in res] == [[2, 5], [2, 5]]
    assert st.calls[-1] == ("search", 2, 2, 50, [0b100100100])
    docs = run(store.query_similar_documents(q, k=2, pages_per_document=2, doc_ids=["d0", "d2"]))
    assert [[c.chunk_number for c in d] for d in docs] == [[0], [2]]
    assert st.calls[-1] == ("search_docs", 2, 2, 50, [0b101101101])
    assert run(store.query_similar(q, k=3, doc_ids=["nope"])) == []


def test_compaction_goes_through_the_sign_stage():
    store = store_with_fake(compact_dead_fraction=0.2)
    emb = np.ones((2, 128), np.float32)
    run(store.store_embeddings([DocumentChunk(document_id=f"d{i % 2}", chunk_number=i, content="", embedding=emb, metadata={})
                                for i in range(6)]))
    assert run(store.delete_chunks_by_document_id("d0"))
    assert ("compact", [1, 3, 5]) in store._two_stage.calls and store._two_stage.n == 3
