"""B200MultiVectorStore.query_similar_with_feedback without a GPU: which chunks become examples and with what weights, the
request mask (the doc_ids / app_id filter minus every example chunk), the both-lists error, min_score, compaction, and the
routing through an injected index (exhaustive) and an injected first stage (two-stage), in the pattern of
test_similar_store_cpu.py.  The stand-in index fuses a fixed oracle score table with the weights it is given, so every
expected list is worked out here."""
import asyncio

import numpy as np
import pytest

from morphik_core_b200.models import DocumentChunk
from morphik_core_b200.store import B200MultiVectorStore

N = 9  # pages 0..8: document d{i % 3}, chunk i


def _allowed(row, n):
    return np.unpackbits(np.asarray(row, np.uint32).view(np.uint8), bitorder="little")[:n].astype(bool)


def oracle(a, b):
    """Stand-in similarity: closer chunk numbers are more alike."""
    return 1.0 / (1.0 + abs(a - b))


def query(chunk):
    """A query embedding the stand-in reads as "like chunk `chunk`"."""
    q = np.zeros((2, 128), np.float32)
    q[0, 0] = chunk
    return q


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

    def search_examples(self, q_dev, q_lens, ex_pages, ex_req, ex_weights, n_req, k, allow_mask_dev=None,
                        mask_index_dev=None):
        import torch

        masks = allow_mask_dev.numpy().view(np.uint32)
        self.calls.append(("search_examples", None if q_dev is None else q_dev.numpy().copy(), list(q_lens),
                           list(ex_pages), list(ex_req), [float(w) for w in ex_weights], n_req, k, masks.copy(),
                           mask_index_dev.tolist()))
        like = [float(q_dev[0, 0])] if q_lens else []
        like += [self.order[p] for p in ex_pages]
        ts = np.full((n_req, k), -np.inf, np.float32)
        ti = np.full((n_req, k), -1, np.int64)
        tc = np.zeros(n_req, np.int32)
        for r in range(n_req):
            ok = np.flatnonzero(_allowed(masks[int(mask_index_dev[r])], self.n))
            sc = np.array([sum(w * oracle(c, self.order[p]) for c, q, w in zip(like, ex_req, ex_weights) if q == r)
                           for p in ok], np.float32)
            order = sorted(range(len(ok)), key=lambda j: (-sc[j], ok[j]))[:k]
            ts[r, :len(order)] = sc[order]
            ti[r, :len(order)] = ok[order]
            tc[r] = len(order)
        return torch.from_numpy(ts), torch.from_numpy(ti), torch.from_numpy(tc)


class FakeStage:
    """The two-stage search with every allowed page a candidate: the rerank is the exhaustive ranking."""

    def __init__(self, index):
        self.index = index
        self.calls = []
        self.last_timing_ms = {}

    def add_pages(self, pages):
        return self.index.add_pages(pages)

    def compact(self, keep):
        self.index.compact(keep)

    def search_examples(self, queries, pages, ex_req, ex_weights, n_req, k, n_candidates=1000, allow_masks=None):
        import torch

        self.calls.append(("search_examples", len(queries), list(pages), k, n_candidates, np.array(allow_masks).shape))
        self.last_timing_ms = {"encode_query_ms": 1.0}
        mat = torch.from_numpy(np.ascontiguousarray(allow_masks, np.uint32).view(np.int32))
        q = torch.from_numpy(np.concatenate(queries)) if queries else None
        ts, ti, tc = (t.numpy() for t in self.index.search_examples(q, [len(x) for x in queries], pages, ex_req, ex_weights,
                                                                    n_req, k, mat, torch.zeros(n_req, dtype=torch.int32)))
        return ts, ti, tc


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
    return [(r.document_id, r.chunk_number) for r in res]


def want(likes, unlikes, pages, k):
    """Expected (document, chunk) list: the allowed pages by mean like minus mean unlike similarity DESC, page ASC."""
    def score(p):
        s = sum(oracle(c, p) for c in likes) / len(likes)
        return s - (sum(oracle(c, p) for c in unlikes) / len(unlikes) if unlikes else 0.0)

    best = sorted(pages, key=lambda p: (-np.float32(score(p)), p))[:k]
    return [(f"d{p % 3}", p) for p in best]


@pytest.mark.parametrize("two_stage", [False, True])
def test_weights_examples_and_mask(two_stage):
    store, idx = _store(two_stage)
    res = run(store.query_similar_with_feedback(query(2), k=4, positive_chunks=[("d0", 3), ("d1", 4)],
                                                negative_chunks=[("d2", 8)]))
    rest = [p for p in range(N) if p not in (3, 4, 8)]
    assert chunks(res) == want([2, 3, 4], [8], rest, 4)
    call = idx.calls[-1]
    assert call[2] == [2] and call[3] == [3, 4, 8] and call[4] == [0, 0, 0, 0] and call[6] == 1 and call[7] == 4
    assert call[5] == pytest.approx([1 / 3, 1 / 3, 1 / 3, -1.0])
    assert _allowed(call[8][0], N).tolist() == [p in rest for p in range(N)]
    if two_stage:
        assert store._two_stage.calls[-1][1:] == (1, [3, 4, 8], 4, 40, (1, 1))
        assert store.last_query_timing["encode_query_ms"] == 1.0
    # no query: the positives alone, each 1/n_pos; two negatives -1/2 each
    run(store.query_similar_with_feedback(None, k=3, positive_chunks=[("d0", 0), ("d1", 1)],
                                          negative_chunks=[("d2", 5), ("d0", 6)]))
    call = idx.calls[-1]
    assert call[1] is None and call[2] == [] and call[3] == [0, 1, 5, 6]
    assert call[5] == pytest.approx([0.5, 0.5, -0.5, -0.5])


@pytest.mark.parametrize("two_stage", [False, True])
def test_visibility_duplicates_and_empty_requests(two_stage):
    store, idx = _store(two_stage)
    res = run(store.query_similar_with_feedback(None, k=2, positive_chunks=[("d1", 7), ("nope", 1), ("d1", 7)],
                                                negative_chunks=[("d2", 99), ("d0", 0), ("d0", 0)]))
    assert chunks(res) == want([7], [0], [p for p in range(N) if p not in (0, 7)], 2)
    assert idx.calls[-1][3] == [7, 0] and idx.calls[-1][5] == pytest.approx([1.0, -1.0])
    n = len(idx.calls)
    # no query and no visible positive: nothing to search
    assert run(store.query_similar_with_feedback(None, k=3, positive_chunks=[("nope", 1)])) == []
    assert run(store.query_similar_with_feedback(None, k=3, negative_chunks=[("d0", 0)])) == []
    assert run(store.query_similar_with_feedback(query(1), k=0)) == []
    assert len(idx.calls) == n
    # a query alone is a plain search
    res = run(store.query_similar_with_feedback(query(4), k=3))
    assert chunks(res) == want([4], [], range(N), 3)


def test_a_chunk_in_both_lists_is_an_error():
    store, idx = _store()
    with pytest.raises(ValueError, match="both"):
        run(store.query_similar_with_feedback(query(1), k=3, positive_chunks=[("d0", 3)], negative_chunks=[("d1", 1), ("d0", 3)]))
    assert idx.calls == []


def test_app_id_scopes_examples_and_results():
    store, idx = _store(app="a")
    run(store.store_embeddings([DocumentChunk(document_id="e", chunk_number=i, content="", embedding=np.ones((2, 128), np.float32),
                                              metadata={}) for i in range(9, 11)], app_id="b"))
    # a positive of another app is skipped: nothing left to search with
    assert run(store.query_similar_with_feedback(None, k=5, positive_chunks=[("e", 9)], app_id="a")) == []
    res = run(store.query_similar_with_feedback(None, k=20, positive_chunks=[("d0", 3)], negative_chunks=[("e", 10)],
                                                app_id="a"))
    assert idx.calls[-1][3] == [3]  # the other app's negative is skipped too
    assert all(d != "e" for d, _ in chunks(res)) and len(res) == N - 1


@pytest.mark.parametrize("two_stage", [False, True])
def test_doc_ids_filter_and_min_score(two_stage):
    store, idx = _store(two_stage)
    res = run(store.query_similar_with_feedback(None, k=9, positive_chunks=[("d0", 3)], doc_ids=["d1", "d0"]))
    assert chunks(res) == want([3], [], [0, 1, 4, 6, 7], 9)
    res = run(store.query_similar_with_feedback(None, k=9, positive_chunks=[("d0", 3)], min_score=0.3))
    assert chunks(res) == want([3], [], [1, 2, 4, 5], 9)  # the others score 0.25 or less
    assert run(store.query_similar_with_feedback(None, k=9, positive_chunks=[("d0", 3)], doc_ids=["nope"])) == []


@pytest.mark.parametrize("two_stage", [False, True])
def test_examples_keep_their_pages_across_compaction(two_stage):
    store, idx = _store(two_stage)
    store.compact_dead_fraction = 0.0
    assert run(store.delete_chunks_by_document_id("d1"))  # compacts at once
    assert idx.n == 6
    assert run(store.query_similar_with_feedback(None, k=5, positive_chunks=[("d1", 4)])) == []
    res = run(store.query_similar_with_feedback(None, k=9, positive_chunks=[("d0", 3), ("d1", 4)],
                                                negative_chunks=[("d2", 5)]))
    assert chunks(res) == want([3], [5], [0, 2, 6, 8], 9)
    assert idx.calls[-1][3] == [2, 3]  # d0 chunk 3 and d2 chunk 5 at their compacted page ids
