"""B200MultiVectorStore.index_duplicates / find_duplicate_chunks / query_similar_distinct without a GPU, through a stand-in
index (the pattern of test_similar_store_cpu.py): the stand-in's pages hold a "content id", pages of equal content id are
duplicates (sim 1 both ways, 0.2 otherwise), and a query scores a page by a fixed table.  Covers masks that never join or
reveal invisible pages, deletion, compaction, pages added after index_duplicates, min_score, k capping, an empty store and
the refusals."""
import asyncio

import numpy as np
import pytest
import torch

from duplicates_oracle import collapsed_topk, union_find_labels
from morphik_core_b200.models import DocumentChunk
from morphik_core_b200.store import B200MultiVectorStore


def _allowed(words, n):
    if words is None:
        return np.ones(n, bool)
    w = np.asarray(words.numpy() if isinstance(words, torch.Tensor) else words).view(np.uint32)
    return np.unpackbits(w.view(np.uint8), bitorder="little")[:n].astype(bool)


class FakeIndex:
    device = "cpu"
    row_bytes = 256

    def __init__(self):
        self.content = []  # page -> content id
        self.calls = []

    @property
    def n(self):
        return len(self.content)

    def add_pages(self, pages):
        first = self.n
        self.content += [int(p[0, 0]) for p in pages]
        return first, len(pages)

    def compact(self, keep):
        self.content = [self.content[p] for p in keep]

    def duplicate_candidates(self, src, n_cand, mask):
        self.calls.append(("candidates", list(src), n_cand))
        ok = _allowed(mask, self.n)
        a, b = [], []
        for s in src:
            for p in [p for p in range(self.n) if ok[p] and p != s][:n_cand]:
                a.append(min(s, p))
                b.append(max(s, p))
        key = sorted(set(zip(a, b)))
        return (torch.tensor([k[0] for k in key], dtype=torch.int64), torch.tensor([k[1] for k in key], dtype=torch.int64))

    def pair_maxsim(self, a, b):
        self.calls.append(("pair_maxsim", a.tolist(), b.tolist()))
        s = torch.tensor([1.0 if self.content[x] == self.content[y] else 0.2 for x, y in zip(a.tolist(), b.tolist())])
        return s, s.clone()

    def duplicate_groups(self, a, b, sab, sba, threshold, mask):
        ok = _allowed(mask, self.n)
        e = [(x, y) for x, y, s, t in zip(a.tolist(), b.tolist(), sab.tolist(), sba.tolist())
             if s >= threshold and t >= threshold and ok[x] and ok[y]]
        return torch.from_numpy(union_find_labels(self.n, e, ok))

    def search_docs(self, queries, k, per, group, n_docs, allow_mask=None):
        assert per == 1 and n_docs == self.n
        scores = np.array([score(c) for c in self.content], np.float64)
        lab = group.numpy().astype(np.int64)
        ok = _allowed(allow_mask, self.n)
        lab[~ok] = -1
        best = collapsed_topk(scores, lab, k)
        ts = np.full((1, k, 1), -np.inf, np.float32)
        ti = np.full((1, k, 1), -1, np.int64)
        pc = np.zeros((1, k), np.int32)
        ts[0, :len(best), 0] = scores[best]
        ti[0, :len(best), 0] = best
        pc[0, :len(best)] = 1
        return ts, ti, pc, np.array([len(best)], np.int32)


def score(content):
    return 10.0 - content  # lower content id ranks higher


def run(coro):
    return asyncio.run(coro)


# page p: document d{p % 3}, content id CONTENT[p]
CONTENT = [0, 1, 0, 2, 3, 1, 4, 0, 5]


def _store(contents=CONTENT, tier="hbm"):
    idx = FakeIndex()
    store = B200MultiVectorStore(auto_initialize=False, index=idx, coalesce_queries=False)
    store.corpus_tier = tier
    _add(store, contents, 0)
    return store, idx


def _add(store, contents, first, app=None):
    run(store.store_embeddings([DocumentChunk(document_id=f"d{(first + i) % 3}", chunk_number=first + i, content="",
                                              embedding=np.full((2, 128), c, np.float32), metadata={})
                                for i, c in enumerate(contents)], app_id=app))


def groups(res):
    return [[c.chunk_number for c in g] for g in res]


def test_groups_and_distinct_search():
    store, _ = _store()
    assert run(store.index_duplicates(n_candidates=8)) > 0
    assert groups(run(store.find_duplicate_chunks(0.5))) == [[0, 2, 7], [1, 5]]
    got = run(store.query_similar_distinct(np.ones((3, 128)), k=4, threshold=0.5))
    assert [c.chunk_number for c in got] == [0, 1, 3, 4]
    assert [c.score for c in got] == [10.0, 9.0, 8.0, 7.0]
    assert sorted(got[0].metadata["duplicates"]) == [("d1", 7), ("d2", 2)]
    assert got[2].metadata["duplicates"] == []
    # a threshold above every sim: no groups, the flat ranking
    assert run(store.find_duplicate_chunks(1.5)) == []
    got = run(store.query_similar_distinct(np.ones((3, 128)), k=3, threshold=1.5))
    assert [c.chunk_number for c in got] == [0, 2, 7]


def test_masks_never_join_or_reveal_invisible_pages():
    store, _ = _store([0, 1, 0, 0, 2, 1])  # 0 - 2 - 3 in d0 / d2 / d0, 1 - 5 in d1 / d2
    run(store.index_duplicates(n_candidates=8))
    # d2 hidden: page 2 and page 5 are invisible, so neither joins anything nor appears as a duplicate
    res = run(store.find_duplicate_chunks(0.5, doc_ids=["d0", "d1"]))
    assert groups(res) == [[0, 3]]
    got = run(store.query_similar_distinct(np.ones((3, 128)), k=5, threshold=0.5, doc_ids=["d0", "d1"]))
    assert [c.chunk_number for c in got] == [0, 1, 4]
    assert [x[1] for x in got[0].metadata["duplicates"]] == [3] and got[1].metadata["duplicates"] == []


def test_a_group_is_not_joined_through_a_hidden_page():
    idx = FakeIndex()
    store = B200MultiVectorStore(auto_initialize=False, index=idx, coalesce_queries=False)
    _add(store, [0, 0], 0)
    _add(store, [0], 2, app="other")  # visible to app "other" only
    # only 0 - 2 and 1 - 2 are pairs: 0 and 1 meet through page 2 alone
    idx.duplicate_candidates = lambda src, n, mask: (torch.tensor([0, 1]), torch.tensor([2, 2]))
    run(store.index_duplicates())
    assert groups(run(store.find_duplicate_chunks(0.5, app_id="other"))) == [[0, 1, 2]]
    assert groups(run(store.find_duplicate_chunks(0.5, app_id="mine"))) == []


def test_deleted_pages_drop_out_and_compaction_remaps():
    store, idx = _store()
    store.compact_dead_fraction = 1.0  # no compaction on delete
    run(store.index_duplicates(n_candidates=8))
    run(store.delete_chunks_by_document_id("d2"))  # pages 2, 5, 8
    assert groups(run(store.find_duplicate_chunks(0.5))) == [[0, 7]]
    n_pairs = len(store._dup["a"])
    with store._lock:
        store._compact_locked()
    # pages 0 1 3 4 6 7 -> 0 1 2 3 4 5; chunk numbers stay
    assert groups(run(store.find_duplicate_chunks(0.5))) == [[0, 7]]
    assert store._dup["n_indexed"] == 6 and len(store._dup["a"]) < n_pairs
    assert int(store._dup["a"].max()) < 6 and int(store._dup["b"].max()) < 6


def test_pages_added_later_stay_singletons_until_the_next_call():
    store, idx = _store()
    run(store.index_duplicates(n_candidates=8))
    _add(store, [1, 3], 9)
    assert groups(run(store.find_duplicate_chunks(0.5))) == [[0, 2, 7], [1, 5]]
    idx.calls.clear()
    run(store.index_duplicates(n_candidates=8))
    assert idx.calls[0] == ("candidates", [9, 10], 8)  # only the new pages are sources
    assert groups(run(store.find_duplicate_chunks(0.5))) == [[0, 2, 7], [1, 5, 9], [4, 10]]
    idx.calls.clear()
    run(store.index_duplicates(n_candidates=8, rebuild=True))
    assert idx.calls[0] == ("candidates", list(range(11)), 8)
    assert groups(run(store.find_duplicate_chunks(0.5))) == [[0, 2, 7], [1, 5, 9], [4, 10]]


def test_min_score_k_cap_and_empty_store():
    store, _ = _store()
    run(store.index_duplicates(n_candidates=8))
    got = run(store.query_similar_distinct(np.ones((3, 128)), k=100, threshold=0.5, min_score=7.5))
    assert [c.chunk_number for c in got] == [0, 1, 3]
    assert len(run(store.query_similar_distinct(np.ones((3, 128)), k=100, threshold=0.5))) == 6
    assert run(store.query_similar_distinct(np.ones((3, 128)), k=0, threshold=0.5)) == []
    empty, _ = _store([])
    assert run(empty.index_duplicates()) == 0
    assert run(empty.find_duplicate_chunks(0.5)) == []
    assert run(empty.query_similar_distinct(np.ones((3, 128)), k=3, threshold=0.5)) == []


def test_refusals():
    store, _ = _store()
    with pytest.raises(RuntimeError):
        run(store.find_duplicate_chunks(0.5))
    with pytest.raises(RuntimeError):
        run(store.query_similar_distinct(np.ones((3, 128)), k=3, threshold=0.5))
    run(store.index_duplicates())
    for bad in (float("nan"), float("inf"), -float("inf")):
        with pytest.raises(ValueError):
            run(store.find_duplicate_chunks(bad))
        with pytest.raises(ValueError):
            run(store.query_similar_distinct(np.ones((3, 128)), k=3, threshold=bad))
    with pytest.raises(ValueError):
        run(store.index_duplicates(n_candidates=0))
    host, _ = _store(tier="host")
    with pytest.raises(ValueError):
        run(host.index_duplicates())
    with pytest.raises(ValueError):
        run(host.find_duplicate_chunks(0.5))
