"""B200MultiVectorStore.query_similar_to_chunks without a GPU: which sources are searched, the per-source masks (the source,
its document, the doc_ids / app_id filter), min_score, compaction, and the routing through an injected index (exhaustive)
and an injected first stage (two-stage), in the pattern of test_mmr_store_cpu.py.  The stand-in index ranks the allowed
pages by a fixed oracle score table, so every expected list is worked out here."""
import asyncio

import numpy as np
import pytest

from morphik_core_b200.models import DocumentChunk
from morphik_core_b200.store import B200MultiVectorStore

N = 9  # pages 0..8: document d{i % 3}, chunk i


def _allowed(row, n):
    return np.unpackbits(np.asarray(row, np.uint32).view(np.uint8), bitorder="little")[:n].astype(bool)


def oracle(src, page):
    """Stand-in similarity: closer chunk numbers are more alike."""
    return 1.0 / (1.0 + abs(src - page))


class FakeIndex:
    row_bytes = 256
    device = "cpu"

    def __init__(self):
        self.n = 0
        self.calls = []
        self.order = []  # page id -> chunk number it holds (changes with compaction)

    def add_pages(self, pages):
        first = self.n
        self.order += list(range(first, first + len(pages)))
        self.n += len(pages)
        return first, len(pages)

    def compact(self, keep):
        self.order = [self.order[p] for p in keep]
        self.n = len(keep)

    def search_pages(self, src_pages, k, allow_mask_dev=None, mask_index_dev=None):
        import torch

        src = [int(p) for p in src_pages]
        masks = allow_mask_dev.numpy().view(np.uint32)
        self.calls.append(("search_pages", src, k, masks.copy(), mask_index_dev.tolist()))
        ts = np.full((len(src), k), -np.inf, np.float32)
        ti = np.full((len(src), k), -1, np.int64)
        tc = np.zeros(len(src), np.int32)
        for i, s in enumerate(src):
            ok = np.flatnonzero(_allowed(masks[int(mask_index_dev[i])], self.n))
            sc = np.array([oracle(self.order[s], self.order[p]) for p in ok], np.float32)
            order = sorted(range(len(ok)), key=lambda j: (-sc[j], ok[j]))[:k]
            ts[i, :len(order)] = sc[order]
            ti[i, :len(order)] = ok[order]
            tc[i] = len(order)
        return torch.from_numpy(ts), torch.from_numpy(ti), torch.from_numpy(tc)


class FakeStage:
    """A first stage of n_candidates pages per source under the masks it is given, then the rerank of those candidates
    (with the stand-in scores, the rerank keeps the first stage's order)."""

    def __init__(self, index):
        self.index = index
        self.calls = []
        self.last_timing_ms = {}

    def add_pages(self, pages):
        return self.index.add_pages(pages)

    def compact(self, keep):
        self.index.compact(keep)

    def search_pages(self, src_pages, k, n_candidates=1000, allow_masks=None):
        import torch

        self.calls.append(("search_pages", list(src_pages), k, n_candidates))
        self.last_timing_ms = {"encode_query_ms": 1.0}
        mat = torch.from_numpy(np.ascontiguousarray(allow_masks, np.uint32).view(np.int32))
        index = torch.arange(len(src_pages), dtype=torch.int32)
        ts, ti, tc = (t.numpy() for t in self.index.search_pages(src_pages, min(n_candidates, self.index.n), mat, index))
        return ts[:, :k], ti[:, :k], np.minimum(tc, k).astype(np.int32)


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
                                              metadata={}) for i in range(N)], app_id=app))
    return store, idx


def chunks(res):
    return [[(r.document_id, r.chunk_number) for r in lst] for lst in res]


def want(src, pages, k):
    """Expected (document, chunk) list: the allowed pages by oracle score DESC, page ASC."""
    best = sorted(pages, key=lambda p: (-oracle(src, p), p))[:k]
    return [(f"d{p % 3}", p) for p in best]


@pytest.mark.parametrize("two_stage", [False, True])
def test_source_and_same_document_are_excluded(two_stage):
    store, idx = _store(two_stage)
    res = run(store.query_similar_to_chunks([("d1", 4)], k=4))
    assert chunks(res) == [want(4, [p for p in range(N) if p % 3 != 1], 4)]
    res = run(store.query_similar_to_chunks([("d1", 4)], k=4, include_same_document=True))
    assert chunks(res) == [want(4, [p for p in range(N) if p != 4], 4)]
    assert res[0][0].score == pytest.approx(0.5)
    if two_stage:
        assert store._two_stage.calls[-1][2:] == (4, 40)
        assert store.last_query_timing["encode_query_ms"] == 1.0


@pytest.mark.parametrize("two_stage", [False, True])
def test_sources_share_one_call_in_first_mention_order(two_stage):
    store, idx = _store(two_stage)
    res = run(store.query_similar_to_chunks([("d2", 8), ("nope", 3), ("d0", 0), ("d2", 8), ("d1", 99)], k=2))
    assert chunks(res) == [want(8, [p for p in range(N) if p % 3 != 2], 2), want(0, [p for p in range(N) if p % 3], 2)]
    calls = [c for c in idx.calls if c[0] == "search_pages"]
    assert len(calls) == 1 and calls[0][1] == [8, 0]
    assert run(store.query_similar_to_chunks([("nope", 1)], k=3)) == []
    assert run(store.query_similar_to_chunks([("d0", 0)], k=0)) == []
    assert run(store.query_similar_to_chunks([], k=3)) == []


@pytest.mark.parametrize("two_stage", [False, True])
def test_doc_ids_filter_and_min_score(two_stage):
    store, idx = _store(two_stage)
    res = run(store.query_similar_to_chunks([("d0", 3)], k=9, doc_ids=["d1", "d0"]))
    assert chunks(res) == [want(3, [1, 4, 7], 9)]
    if two_stage:  # the first stage gets the source's own row: the filter and the exclusions
        masks = [c for c in idx.calls if c[0] == "search_pages"][-1][3]
        assert _allowed(masks[0], N).tolist() == [p % 3 == 1 for p in range(N)]
    res = run(store.query_similar_to_chunks([("d0", 3)], k=9, min_score=0.3))
    assert chunks(res) == [want(3, [1, 2, 4, 5], 9)]  # the others score 0.25 or less
    assert run(store.query_similar_to_chunks([("d0", 3)], k=9, doc_ids=["d0"])) == [[]]
    assert run(store.query_similar_to_chunks([("d0", 3)], k=9, doc_ids=["nope"])) == [[]]


def test_app_id_scopes_sources_and_results():
    store, idx = _store(app="a")
    run(store.store_embeddings([DocumentChunk(document_id="e", chunk_number=i, content="", embedding=np.ones((2, 128), np.float32),
                                              metadata={}) for i in range(9, 11)], app_id="b"))
    assert run(store.query_similar_to_chunks([("e", 9)], k=5, app_id="a")) == []  # a source of another app is skipped
    res = run(store.query_similar_to_chunks([("d0", 3), ("e", 9)], k=20, app_id="a"))
    assert len(res) == 1 and all(d != "e" for d, _ in chunks(res)[0])
    # the chunks stored under "a" are not visible to "b": only e's own other chunk is left
    assert run(store.query_similar_to_chunks([("e", 9)], k=20, app_id="b")) == [[]]
    res = run(store.query_similar_to_chunks([("e", 9)], k=20, app_id="b", include_same_document=True))
    assert chunks(res) == [[("e", 10)]]


@pytest.mark.parametrize("two_stage", [False, True])
def test_deleted_sources_are_skipped_before_and_after_compaction(two_stage):
    store, idx = _store(two_stage)
    store.compact_dead_fraction = 0.5  # one document of three: tombstoned, not yet compacted
    assert run(store.delete_chunks_by_document_id("d1"))
    assert idx.n == N
    assert run(store.query_similar_to_chunks([("d1", 4)], k=5)) == []
    res = run(store.query_similar_to_chunks([("d0", 3), ("d1", 4)], k=9))
    assert chunks(res) == [want(3, [p for p in range(N) if p % 3 == 2], 9)]
    store.compact_dead_fraction = 0.0
    assert run(store.delete_chunks_by_document_id("none"))  # compacts now
    assert idx.n == 6
    res = run(store.query_similar_to_chunks([("d0", 3), ("d1", 4), ("d2", 5)], k=9))
    assert chunks(res) == [want(3, [2, 5, 8], 9), want(5, [0, 3, 6], 9)]
    calls = [c for c in idx.calls if c[0] == "search_pages"]
    assert calls[-1][1] == [2, 3]  # d0 chunk 3 and d2 chunk 5 at their compacted page ids


@pytest.mark.parametrize("two_stage", [False, True])
def test_a_long_source_document_leaves_k_results_from_other_documents(two_stage):
    """The source's document has more chunks than the first stage has candidate slots, and they are the source's nearest
    pages: the candidates must still be other documents' chunks, so k of them come back."""
    idx = FakeIndex()
    kw = {"fde_candidates": 3} if two_stage else {}
    store = B200MultiVectorStore(auto_initialize=False, index=idx, coalesce_queries=False, **kw)
    if two_stage:
        store._two_stage = FakeStage(idx)
    emb = np.ones((3, 128), np.float32)
    docs = ["big"] * 8 + ["x", "y", "z", "x"]  # chunk i of document docs[i]; "big" holds the 7 chunks nearest to chunk 0
    run(store.store_embeddings([DocumentChunk(document_id=d, chunk_number=i, content="", embedding=emb, metadata={})
                                for i, d in enumerate(docs)]))
    res = run(store.query_similar_to_chunks([("big", 0)], k=3))
    assert chunks(res) == [[("x", 8), ("y", 9), ("z", 10)]]
    res = run(store.query_similar_to_chunks([("big", 0)], k=3, include_same_document=True))
    assert chunks(res) == [[("big", 1), ("big", 2), ("big", 3)]]
