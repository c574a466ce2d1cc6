"""B200MultiVectorStore.query_similar_documents(score_by="document") without a GPU: the filters, app_id, deleted documents,
the evidence-to-chunk mapping, min_score and empty results, routed through an injected index (exhaustive) and an
injected first stage (two-stage), in the pattern of test_similar_store_cpu.py.  The stand-in index scores a page's tokens
from a fixed table of its chunk number and ranks documents with doc_maxsim_oracle, so every expected list is worked out
here."""
import asyncio

import numpy as np
import pytest

from doc_maxsim_oracle import doc_maxsim_np
from morphik_core_b200.models import DocumentChunk
from morphik_core_b200.store import DOCUMENT_SCORE_KEY, B200MultiVectorStore

N = 9  # pages 0..8: document d{i % 3}, chunk i


def token_maxima(chunk):
    """Stand-in per-token maxima of the query's two tokens on the page holding `chunk`."""
    return [float(chunk), float(chunk * 5 % 9)]


def _allowed(words, n):
    if words is None:
        return np.ones(n, bool)
    return np.unpackbits(np.asarray(words, np.uint32).view(np.uint8), bitorder="little")[:n].astype(bool)


class FakeIndex:
    row_bytes = 256
    device = "cpu"
    tier = "hbm"

    def __init__(self):
        self.n = 0
        self.calls = []
        self.order = []  # page id -> chunk number it holds

    def add_pages(self, pages):
        first = self.n
        self.order += list(range(first, first + len(pages)))
        self.n += len(pages)
        return first, len(pages)

    def compact(self, keep):
        self.order = [self.order[p] for p in keep]
        self.n = len(keep)

    def search_doc_maxsim(self, queries, k, per_doc, page_doc_dev, n_docs, allow_mask=None):
        self.calls.append(("search_doc_maxsim", k, per_doc, n_docs))
        m = np.array([token_maxima(c) for c in self.order])
        page_doc = page_doc_dev.numpy()
        docs, S, ev = doc_maxsim_np(m, page_doc, n_docs, k, per_doc, counted=_allowed(allow_mask, self.n))
        ds = np.full((1, k), -np.inf, np.float32)
        di = np.full((1, k), -1, np.int64)
        ei = np.full((1, k, per_doc), -1, np.int64)
        es = np.full((1, k, per_doc), -np.inf, np.float32)
        ec = np.zeros((1, k), np.int32)
        ds[0, :len(docs)], di[0, :len(docs)] = S, docs
        for i, (pages, shares) in enumerate(ev):
            ei[0, i, :len(pages)], es[0, i, :len(pages)], ec[0, i] = pages, shares, len(pages)
        return ds, di, ei, es, ec, np.array([len(docs)], np.int32)


class FakeStage:
    def __init__(self, index):
        self.index = index
        self.calls = []
        self.last_timing_ms = {}

    def add_pages(self, pages):
        return self.index.add_pages(pages)

    def compact(self, keep):
        self.index.compact(keep)

    def search_doc_maxsim(self, queries, k, per_doc, page_doc_dev, n_docs, n_candidates=1000, allow_mask=None):
        self.calls.append(("search_doc_maxsim", k, per_doc, n_candidates))
        return self.index.search_doc_maxsim(queries, k, per_doc, page_doc_dev, n_docs, allow_mask)


def run(coro):
    return asyncio.run(coro)


def _store(two_stage=False, app=None):
    idx = FakeIndex()
    kw = {"fde_candidates": 40} if two_stage else {}
    store = B200MultiVectorStore(auto_initialize=False, index=idx, coalesce_queries=False, **kw)
    if two_stage:
        store._two_stage = FakeStage(idx)
    emb = np.ones((3, 128), np.float32)
    run(store.store_embeddings([DocumentChunk(document_id=f"d{i % 3}", chunk_number=i, content=str(i), embedding=emb,
                                              metadata={"i": i}) for i in range(N)], app_id=app))
    return store, idx


def query(store, k=5, per=4, **kw):
    return run(store.query_similar_documents(np.ones((2, 128), np.float32), k, pages_per_document=per, score_by="document",
                                             **kw))


def shape(res):
    """[(document, document score, [(chunk, share), ...]), ...]"""
    out = []
    for lst in res:
        assert len({c.metadata[DOCUMENT_SCORE_KEY] for c in lst}) == 1
        out.append((lst[0].document_id, lst[0].metadata[DOCUMENT_SCORE_KEY], [(c.chunk_number, c.score) for c in lst]))
    return out


# token maxima per chunk: 0 [0,0] 1 [1,5] 2 [2,1] 3 [3,6] 4 [4,2] 5 [5,7] 6 [6,3] 7 [7,8] 8 [8,4]
# d0 (0, 3, 6): [6 @6, 6 @3] = 12;  d1 (1, 4, 7): [7 @7, 8 @7] = 15;  d2 (2, 5, 8): [8 @8, 7 @5] = 15
FULL = [("d1", 15.0, [(7, 15.0)]), ("d2", 15.0, [(8, 8.0), (5, 7.0)]), ("d0", 12.0, [(3, 6.0), (6, 6.0)])]


@pytest.mark.parametrize("two_stage", [False, True])
def test_documents_rank_by_their_pooled_tokens_with_evidence_chunks(two_stage):
    store, idx = _store(two_stage)
    res = query(store)
    assert shape(res) == FULL
    assert res[0][0].metadata["i"] == 7  # the chunk's own metadata is kept
    assert shape(query(store, k=2, per=1)) == [("d1", 15.0, [(7, 15.0)]), ("d2", 15.0, [(8, 8.0)])]
    if two_stage:
        assert store._two_stage.calls[-1] == ("search_doc_maxsim", 2, 1, 40)
    else:
        assert idx.calls[-1] == ("search_doc_maxsim", 2, 1, 3)


@pytest.mark.parametrize("two_stage", [False, True])
def test_doc_ids_filter_and_min_score(two_stage):
    store, _ = _store(two_stage)
    assert shape(query(store, doc_ids=["d0", "d2"])) == [FULL[1], FULL[2]]
    assert shape(query(store, min_score=13.0)) == FULL[:2]
    assert shape(query(store, min_score=15.0)) == FULL[:2]
    assert query(store, min_score=16.0) == []
    assert query(store, doc_ids=["nope"]) == []
    assert query(store, doc_ids=[]) == []
    assert query(store, k=0) == []


def test_app_id_scopes_the_documents():
    store, idx = _store(app="a")
    emb = np.ones((2, 128), np.float32)
    run(store.store_embeddings([DocumentChunk(document_id="e", chunk_number=i, content="", embedding=emb, metadata={})
                                for i in range(9, 11)], app_id="b"))
    # chunks 9 and 10: [9, 0] and [10, 5] -> e = 10 + 5 = 15, d1's tie, but a later ordinal
    assert shape(query(store, app_id="a")) == FULL
    assert shape(query(store, app_id="b")) == [("e", 15.0, [(10, 15.0)])]
    assert [d for d, _, _ in shape(query(store))] == ["d1", "d2", "e", "d0"]


@pytest.mark.parametrize("two_stage", [False, True])
def test_deleted_documents_do_not_count_before_and_after_compaction(two_stage):
    store, idx = _store(two_stage)
    store.compact_dead_fraction = 0.5  # tombstoned, not yet compacted
    assert run(store.delete_chunks_by_document_id("d1"))
    assert idx.n == N
    assert shape(query(store)) == [FULL[1], FULL[2]]
    store.compact_dead_fraction = 0.0
    assert run(store.delete_chunks_by_document_id("none"))  # compacts now
    assert idx.n == 6
    assert shape(query(store)) == [FULL[1], FULL[2]]


def test_score_by_is_checked_and_page_stays_the_default():
    store, idx = _store()
    with pytest.raises(ValueError, match="score_by"):
        run(store.query_similar_documents(np.ones((2, 128), np.float32), 3, score_by="pages"))
    assert run(store.query_similar_documents(np.ones((2, 128), np.float32), 0)) == []
    assert not idx.calls


def test_an_empty_store_returns_nothing():
    store = B200MultiVectorStore(auto_initialize=False, index=FakeIndex(), coalesce_queries=False)
    assert query(store) == []
