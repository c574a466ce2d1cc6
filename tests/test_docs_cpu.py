"""Grouping results by document without a GPU: the numpy oracle (tests/docs_oracle.py) against an independent walk of the
flat ranking, PageCatalog's page -> document column across add / delete / compaction, and
B200MultiVectorStore.query_similar_documents' host logic with an injected index whose grouped results come from the oracle."""
import asyncio
import functools
import math

import numpy as np
import pytest
import torch

from docs_oracle import topk_docs_np
from morphik_core_b200.catalog import PageCatalog, PageRecord
from morphik_core_b200.models import DocumentChunk
from morphik_core_b200.store import B200MultiVectorStore
from oracle import maxsim_oracle as orc


def _before(a, b):
    """Python restatement of the flat order on (score, id) pairs: NaN first (tied), then score DESC, -0 == +0, id ASC."""
    (sa, ia), (sb, ib) = a, b
    na, nb = math.isnan(sa), math.isnan(sb)
    if na != nb:
        return -1 if na else 1
    if not na and sa != sb:
        return -1 if sa > sb else 1
    return -1 if ia < ib else (1 if ia > ib else 0)


def walk(scores, page_doc, n_docs, k, per_doc, allow=None, cand=None):
    """The contract read literally: rank every eligible item, then walk the ranking."""
    n = len(scores)
    pages = list(range(n)) if cand is None else [int(c) for c in cand]
    seen, items = set(), []
    for j in range(n):
        p = pages[j]
        if not 0 <= p < len(page_doc) or not 0 <= page_doc[p] < n_docs or (allow is not None and not allow[p]):
            continue
        if p in seen:  # candidate mode: a page counts once, at its earliest slot
            continue
        seen.add(p)
        items.append((float(scores[j]), j))
    items.sort(key=functools.cmp_to_key(_before))
    docs = {}
    for _, j in items:
        d = int(page_doc[pages[j]])
        if d not in docs and len(docs) < k:
            docs[d] = []
        if d in docs and len(docs[d]) < per_doc:
            docs[d].append(j)
    return list(docs.values())


def _values(rng, n):
    pool = np.asarray([0.5, 0.25, 0.0, -0.0, 1.0, np.inf, -np.inf, np.nan, -2.0], np.float32)
    v = rng.standard_normal(n).astype(np.float32)
    m = rng.random(n) < 0.6
    v[m] = rng.choice(pool, size=int(m.sum()))
    return v


@pytest.mark.parametrize("seed", range(12))
def test_oracle_equals_walking_the_flat_ranking(seed):
    rng = np.random.default_rng(seed)
    n = int(rng.integers(1, 400))
    n_docs = int(rng.integers(1, n + 1))
    page_doc = rng.integers(0, n_docs, size=n).astype(np.int32)
    page_doc[rng.random(n) < 0.1] = -1
    page_doc[rng.random(n) < 0.05] = n_docs + 3
    if seed % 3 == 0:
        page_doc = np.sort(page_doc)  # contiguous documents, holes first
    k, per_doc = int(rng.integers(1, n_docs + 3)), int(rng.integers(1, 6))
    allow = rng.random(n) < 0.8 if seed % 2 else None
    cand = None
    if seed % 4 == 1:  # candidate lists: unused slots, ids past the corpus, repeated pages
        m = int(rng.integers(1, 2 * n))
        cand = rng.integers(-1, n + 3, size=m)
        cand[rng.integers(0, m, size=m // 4)] = cand[rng.integers(0, m, size=m // 4)]
        allow = None
    scores = _values(rng, n if cand is None else len(cand))
    if seed % 4 == 1:  # a page has one score, whichever slot holds it
        by_page = _values(rng, n + 3)
        scores = np.where(cand >= 0, by_page[np.maximum(cand, 0)], scores).astype(np.float32)
    pos, ids, counts, nd = topk_docs_np(scores, page_doc, n_docs, k, per_doc, allow=allow, cand=cand)
    want = walk(scores, page_doc, n_docs, k, per_doc, allow=allow, cand=cand)
    assert nd == len(want)
    pages = np.arange(len(scores)) if cand is None else cand
    for r in range(k):
        got = [int(x) for x in pos[r, :counts[r]]]
        assert got == (want[r] if r < nd else [])
        assert ids[r, :counts[r]].tolist() == [int(pages[j]) for j in got]
        assert (pos[r, counts[r]:] == -1).all() and (ids[r, counts[r]:] == -1).all()


def test_oracle_identity_grouping_is_the_flat_topk():
    rng = np.random.default_rng(3)
    s = _values(rng, 500)
    allow = rng.random(500) < 0.7
    for k in (1, 17, 600):
        ts, ti = orc.topk_np(s, k, allow)
        pos, ids, counts, nd = topk_docs_np(s, np.arange(500, dtype=np.int32), 500, k, 1, allow=allow)
        assert nd == len(ti) and ids[:nd, 0].tolist() == ti.tolist() and counts.tolist() == [1] * nd + [0] * (k - nd)


def test_oracle_int32_sums_past_2_24():
    s = np.asarray([(1 << 25) + 1, 1 << 25, (1 << 25) + 1, 5], np.int64)  # equal as float32, distinct as integers
    pos, ids, counts, nd = topk_docs_np(s, np.asarray([0, 1, 1, 2], np.int32), 3, 3, 2)
    assert nd == 3 and pos[0, 0] == 0 and pos[1].tolist() == [2, 1] and pos[2, 0] == 3


def test_catalog_page_documents_across_delete_and_compaction():
    cat = PageCatalog()
    assert cat.page_documents().tolist() == [] and cat.n_documents == 0
    for d, n in [("a", 0), ("b", 0), ("a", 1), ("c", 0), ("b", 1), ("c", 1)]:
        cat.add(PageRecord(d, n, f"{d}{n}", {}))
    assert cat.page_documents().tolist() == [0, 1, 0, 2, 1, 2] and cat.n_documents == 3
    assert cat.page_documents().dtype == np.int32
    cat.delete_document("a")
    assert cat.page_documents().tolist() == [-1, 1, -1, 2, 1, 2] and cat.n_documents == 3
    cat.add(PageRecord("d", 0, "d0", {}))
    assert cat.page_documents().tolist() == [-1, 1, -1, 2, 1, 2, 3] and cat.n_documents == 4
    keep, _ = cat.compaction_plan()
    cat.apply_compaction(keep)  # renumbers the documents in order of their first surviving page
    assert cat.page_documents().tolist() == [0, 1, 0, 1, 2] and cat.n_documents == 3
    assert [cat.records[p].document_id for p in range(5)] == ["b", "c", "b", "c", "d"]


# ------------------------------------------------------------------------------------------------ store host logic
class DocsOracleIndex:
    """Stands in for MaxSimIndex: float MaxSim in float64, grouped by the oracle."""

    row_bytes = 256
    device = torch.device("cpu")

    def __init__(self):
        self.pages = []
        self.calls = []

    def add_pages(self, pages):
        first = len(self.pages)
        self.pages.extend(np.asarray(p, np.float32) for p in pages)
        return first, len(pages)

    def compact(self, keep):
        self.pages = [self.pages[int(i)] for i in keep]

    def search_docs(self, queries, k, per_doc, page_doc_dev, n_docs, allow_mask=None):
        page_doc = page_doc_dev.numpy()
        assert page_doc.shape == (len(self.pages),) and n_docs <= len(self.pages)
        self.calls.append((k, per_doc, n_docs, page_doc_dev))
        allow = None
        if allow_mask is not None:
            allow = np.unpackbits(allow_mask.view(np.uint8), bitorder="little")[: len(self.pages)].astype(bool)
        out = (np.full((len(queries), k, per_doc), -np.inf, np.float32), np.full((len(queries), k, per_doc), -1, np.int64),
               np.zeros((len(queries), k), np.int32), np.zeros(len(queries), np.int32))
        for qi, q in enumerate(queries):
            s = np.asarray([(q.astype(np.float64) @ p.T.astype(np.float64)).max(axis=1).sum() for p in self.pages], np.float32)
            pos, ids, counts, nd = topk_docs_np(s, page_doc, n_docs, k, per_doc, allow=allow)
            out[0][qi] = np.where(pos >= 0, s[np.maximum(pos, 0)], -np.inf)
            out[1][qi], out[2][qi], out[3][qi] = ids, counts, nd
        return out


def _run(coro):
    return asyncio.run(coro)


def _store():
    rng = np.random.default_rng(9)
    idx = DocsOracleIndex()
    store = B200MultiVectorStore(mode="bf16", auto_initialize=False, index=idx, compact_dead_fraction=0.5)
    chunks = []
    for d, n in [("a", 3), ("b", 1), ("c", 4), ("d", 2)]:
        for c in range(n):
            chunks.append(DocumentChunk(document_id=d, chunk_number=c, content=f"{d}{c}", metadata={"m": c},
                                        embedding=rng.standard_normal((5, 128)).astype(np.float32)))
    _run(store.store_embeddings(chunks[:6], app_id="app1"))
    _run(store.store_embeddings(chunks[6:]))
    q = chunks[4].embedding[:3] + 0.01  # closest to c1
    return store, idx, q


def _flat(store, idx, q, **kw):
    """Every chunk by score (float64 MaxSim), grouped by hand."""
    n = len(store.catalog)
    s = np.asarray([(q.astype(np.float64) @ p.T.astype(np.float64)).max(axis=1).sum() for p in idx.pages], np.float32)
    order = orc.rank_desc_np(s, np.arange(n))
    return [(store.catalog.records[p].document_id, store.catalog.records[p].chunk_number, float(s[p])) for p in order
            if store.catalog.alive[p]]


def _key(groups):
    return [[(c.document_id, c.chunk_number, c.score) for c in g] for g in groups]


def test_store_maps_ids_to_chunks_grouped_by_document():
    store, idx, q = _store()
    flat = _flat(store, idx, q)
    got = _run(store.query_similar_documents(q, 2, pages_per_document=2))
    want, seen = [], {}
    for d, c, s in flat:
        if d not in seen and len(seen) < 2:
            seen[d] = len(want)
            want.append([])
        if d in seen and len(want[seen[d]]) < 2:
            want[seen[d]].append((d, c, s))
    assert _key(got) == want and got[0][0].document_id == "c"
    assert got[0][0].content == f"c{got[0][0].chunk_number}" and got[0][0].metadata == {"m": got[0][0].chunk_number}
    assert idx.calls[-1][:3] == (2, 2, 4)
    everything = _run(store.query_similar_documents(q, 50, pages_per_document=64))  # k > number of documents
    assert idx.calls[-1][0] == 4 and len(everything) == 4
    assert sorted((c.document_id, c.chunk_number) for g in everything for c in g) == sorted((d, c) for d, c, _ in flat)
    assert _run(store.query_similar_documents(q, 0)) == []
    with pytest.raises(ValueError):
        _run(store.query_similar_documents(q, 3, pages_per_document=65))


def test_store_filters_min_score_and_caches_the_table():
    store, idx, q = _store()
    got = _run(store.query_similar_documents(q, 4, doc_ids=["a", "d", "zzz"]))
    assert {g[0].document_id for g in got} == {"a", "d"}
    got = _run(store.query_similar_documents(q, 4, app_id="other"))  # chunks stored under app1 are invisible
    assert {g[0].document_id for g in got} == {"c", "d"}
    assert _run(store.query_similar_documents(q, 4, doc_ids=[])) == []
    scores = sorted((c.score for g in _run(store.query_similar_documents(q, 4, pages_per_document=4)) for c in g), reverse=True)
    thr = scores[3]
    got = _run(store.query_similar_documents(q, 4, pages_per_document=4, min_score=thr))
    assert sum(len(g) for g in got) == 4 and all(g and all(c.score >= thr for c in g) for g in got)
    tables = {id(c[3]) for c in idx.calls}
    assert len(tables) == 1  # one device table while the catalogue does not change
    _run(store.delete_chunks_by_document_id("c"))  # 4 of 10 pages dead: below 0.5, no compaction
    got = _run(store.query_similar_documents(q, 4))
    assert "c" not in {g[0].document_id for g in got} and idx.calls[-1][3].tolist()[4:8] == [-1] * 4
    _run(store.delete_chunks_by_document_id("a"))  # 7 of 10 dead: compaction renumbers pages and documents
    assert len(store.catalog) == 3
    got = _run(store.query_similar_documents(q, 4, pages_per_document=3))
    assert sorted(g[0].document_id for g in got) == ["b", "d"] and idx.calls[-1][3].tolist() == [0, 1, 1]


def test_store_empty():
    store = B200MultiVectorStore(mode="bf16", auto_initialize=False, index=DocsOracleIndex())
    q = np.ones((2, 128), np.float32)
    assert _run(store.query_similar_documents(q, 5)) == []
