"""The top k documents instead of the top k pages on an H100 (run with -m gpu): b200ms_topk_docs,
b200ms_search_docs_device, b200ms_rerank_docs_batch_device and B200MultiVectorStore.query_similar_documents.

The grouped result is a pure function of the flat ranking, so every check is exact: ids, counts and score bits.
  - b200ms_topk_docs on crafted matrices (F32 and I32, I32 sums past +-2^31, ties, NaN, +-0, +-inf, out-of-range page_doc,
    an allow mask, one document, k > n_docs, per_doc > pages per document, n_pages > 8192 with a k that slices) against
    tests/docs_oracle.py, and the identity grouping against b200ms_topk;
  - full scans of every corpus dtype against host grouping of the GPU's own flat ranking, unmasked, with one mask, with
    per-query masks, with zero_pad_compat; above 8192 pages against grouping of score_groups' float32 sums;
  - per-query candidate lists with unused slots, ids past the corpus and repeated pages against grouping of
    rerank_batch_device's ranking (a page counts once, at its earliest slot), host tier == HBM tier;
  - refusals launch nothing;
  - the store's query_similar_documents against grouping of query_similar_batch, also after a compaction.
"""
import asyncio
import ctypes

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

torch = pytest.importorskip("torch")
if not torch.cuda.is_available():  # pragma: no cover - the gpu marker normally deselects these on CPU boxes
    pytest.skip("CUDA device required", allow_module_level=True)

from docs_oracle import topk_docs_np  # noqa: E402
from morphik_core_b200 import _native as nat  # noqa: E402
from morphik_core_b200.index import MaxSimIndex  # noqa: E402
from morphik_core_b200.models import DocumentChunk  # noqa: E402
from morphik_core_b200.store import B200MultiVectorStore  # noqa: E402
from oracle.scoring import i32_sum  # noqa: E402

F32 = np.float32
INT_MAX = (1 << 31) - 1
CANON_NAN = np.uint32(0x7FFFFFFF)
EINVAL, ESTATE = -1, -3


def vp(t):
    return ctypes.c_void_p(t.data_ptr()) if t is not None else None


def stream():
    return ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)


def bits_of(x):
    x = np.asarray(x, F32)
    b = x.view(np.uint32).copy()
    b[np.isnan(x)] = CANON_NAN
    return b


def assert_same(got, want, what=""):
    """(scores, ids, page_counts, doc_counts) tuples of numpy arrays: equal bit for bit."""
    gs, gi, gp, gd = got
    ws, wi, wp, wd = want
    assert np.array_equal(gd, wd), (what, gd, wd)
    assert np.array_equal(gp, wp), what
    assert np.array_equal(gi, wi), what
    assert np.array_equal(bits_of(gs), bits_of(ws)), what


def group_flat(scores, ids, count, page_doc, n_docs, k, per_doc, id_base=0):
    """Host grouping of ONE query's flat ranking (scores / ids in rank order, `count` valid): documents by first page,
    their first per_doc pages; a page seen before (a repeated candidate) is skipped."""
    out_s = np.full((k, per_doc), -np.inf, F32)
    out_i = np.full((k, per_doc), -1, np.int64)
    pc = np.zeros(k, np.int32)
    rank, seen = {}, set()
    for s, p in zip(scores[:count], ids[:count]):
        p = int(p)
        if p in seen:
            continue
        seen.add(p)
        d = int(page_doc[p - id_base])
        if not 0 <= d < n_docs:
            continue
        if d not in rank:
            if len(rank) == k:
                continue
            rank[d] = len(rank)
        r = rank[d]
        if pc[r] < per_doc:
            out_s[r, pc[r]], out_i[r, pc[r]] = s, p
            pc[r] += 1
    return out_s, out_i, pc, len(rank)


def stack_expected(rows):
    return (np.stack([r[0] for r in rows]), np.stack([r[1] for r in rows]), np.stack([r[2] for r in rows]),
            np.asarray([r[3] for r in rows], np.int32))


def to_host(t):
    return tuple(x.cpu().numpy() for x in t)


# ------------------------------------------------------------------------------------------------ 1. crafted matrices
def f32_values(rng, shape):
    pool = np.asarray([0.5, 0.25, 0.0, -0.0, 1.0, -1.0, np.inf, -np.inf, np.nan, 3.0], F32)
    v = rng.standard_normal(shape).astype(F32)
    m = rng.random(shape) < 0.6
    v[m] = rng.choice(pool, size=int(m.sum()))
    return v


def i32_values(rng, shape):
    """Group scores whose sums over 2 or 3 groups pass +-2^31, land on +-(2^31 - 1), one past it and next to it."""
    pool = np.asarray([0, 1, -1, 1 << 26, (1 << 26) + 1, -(1 << 27), INT_MAX, INT_MAX - 1, -INT_MAX, -(1 << 31), 1 << 30],
                      np.int64)
    v = rng.integers(-(1 << 28), 1 << 28, size=shape, dtype=np.int64)
    m = rng.random(shape) < 0.6
    v[m] = rng.choice(pool, size=int(m.sum()))
    return v.astype(np.int32)


def doc_table(rng, n_pages, layout):
    """page_doc for a layout: 'runs' (contiguous documents of 1-40 pages, some holes), 'shuffled', 'one' (a single
    document), 'identity' (one page per document)."""
    if layout == "identity":
        return np.arange(n_pages, dtype=np.int32), n_pages
    if layout == "one":
        pd = np.zeros(n_pages, np.int32)
        pd[rng.random(n_pages) < 0.05] = -1
        return pd, 1
    sizes = []
    while sum(sizes) < n_pages:
        sizes.append(int(rng.integers(1, 41)))
    pd = np.repeat(np.arange(len(sizes), dtype=np.int32), sizes)[:n_pages]
    n_docs = int(pd.max()) + 1
    if layout == "shuffled":
        pd = rng.permutation(pd)
    holes = rng.random(n_pages)
    pd[holes < 0.03] = -1
    pd[(holes >= 0.03) & (holes < 0.05)] = n_docs + 7  # >= n_docs: never returned
    return pd.astype(np.int32), n_docs


def topk_docs_raw(h, gs, sdt, n_pages, goff, allow_words, page_doc, n_docs, k, per_doc, scale, id_base):
    n_q = len(goff) - 1
    ts = torch.empty((n_q, k, per_doc), dtype=torch.float32, device="cuda")
    ti = torch.empty((n_q, k, per_doc), dtype=torch.int64, device="cuda")
    pc = torch.empty((n_q, k), dtype=torch.int32, device="cuda")
    dc = torch.empty((n_q,), dtype=torch.int32, device="cuda")
    pd = torch.from_numpy(page_doc).cuda()
    am = None if allow_words is None else torch.from_numpy(allow_words.view(np.int32)).cuda()
    h.check(nat.lib.b200ms_topk_docs(h.ptr, vp(gs), sdt, n_pages, gs.shape[1], nat.i32_array(goff), n_q, vp(am), vp(pd),
                                     int(n_docs), int(k), int(per_doc), ctypes.c_float(scale), int(id_base), vp(ts), vp(ti),
                                     vp(pc), vp(dc), stream()), "b200ms_topk_docs")
    torch.cuda.synchronize()
    return to_host((ts, ti, pc, dc))


def mask_words(allow):
    pad = (-len(allow)) % 32
    bits = np.concatenate([allow, np.zeros(pad, bool)])
    return np.packbits(bits.reshape(-1, 32), axis=1, bitorder="little").view(np.uint32).reshape(-1).copy()


CRAFTED = [  # (n_pages, layout, k, per_doc, masked)
    (100, "runs", 10, 3, False),
    (100, "runs", 50, 64, True),     # k > n_docs, per_doc > pages per document
    (777, "shuffled", 40, 2, True),
    (3000, "one", 5, 4, False),      # one document (and a few holes)
    (1000, "identity", 300, 1, True),
    (20000, "runs", 1000, 2, False),  # > 8192 pages: launch_topk slices (2 slices) and merges
    (70000, "shuffled", 2049, 1, True),
    (70000, "one", 3, 64, False),
]


@pytest.mark.parametrize("sdt", [nat.F32, nat.I32], ids=["f32", "i32"])
@pytest.mark.parametrize("case", CRAFTED, ids=[f"{c[0]}-{c[1]}-k{c[2]}-m{c[3]}{'-mask' if c[4] else ''}" for c in CRAFTED])
def test_topk_docs_against_the_oracle(sdt, case):
    n_pages, layout, k, per_doc, masked = case
    rng = np.random.default_rng(n_pages + k + sdt)
    h = nat.Handle(0)
    groups = [1, 3, 2]
    goff = np.concatenate([[0], np.cumsum(groups)]).astype(np.int32)
    ld = n_pages + 37
    gp = (goff[-1] + 3) // 4 * 4
    vals = f32_values(rng, (gp, ld)) if sdt == nat.F32 else i32_values(rng, (gp, ld))
    page_doc, n_docs = doc_table(rng, n_pages, layout)
    allow = rng.random(n_pages) < 0.7 if masked else None
    scale = 0.5 if sdt == nat.F32 else 1.0 / (127 * 127)
    id_base = 1 << 40
    gs = torch.from_numpy(vals).cuda()
    np.seterr(invalid="ignore", over="ignore")  # inf - inf sums
    got = topk_docs_raw(h, gs, sdt, n_pages, goff, None if allow is None else mask_words(allow), page_doc, n_docs, k,
                        per_doc, scale, id_base)
    want = []
    for q in range(len(groups)):
        if sdt == nat.F32:
            acc = np.zeros(n_pages, F32)
            for g in range(goff[q], goff[q + 1]):
                acc = (acc + vals[g, :n_pages]).astype(F32)
            rep = (acc * F32(scale)).astype(F32)
        else:
            acc = i32_sum(vals[goff[q]:goff[q + 1], :n_pages].astype(np.int64).sum(axis=0))  # the I32 sum rule
            rep = (acc.astype(F32) * F32(scale)).astype(F32)
        pos, ids, pc, nd = topk_docs_np(acc, page_doc, n_docs, k, per_doc, allow=allow)
        sc = np.where(pos >= 0, rep[np.maximum(pos, 0)], F32(-np.inf)).astype(F32)
        want.append((sc, np.where(ids >= 0, ids + id_base, -1), pc, nd))
    assert_same(got, stack_expected(want), case)
    if layout == "identity":  # per_doc == 1 over one page per document: exactly b200ms_topk
        ts = torch.empty((len(groups), k), dtype=torch.float32, device="cuda")
        ti = torch.empty((len(groups), k), dtype=torch.int64, device="cuda")
        tc = torch.empty((len(groups),), dtype=torch.int32, device="cuda")
        am = None if allow is None else torch.from_numpy(mask_words(allow).view(np.int32)).cuda()
        h.check(nat.lib.b200ms_topk(h.ptr, vp(gs), sdt, n_pages, ld, nat.i32_array(goff), len(groups), vp(am), k,
                                    ctypes.c_float(scale), id_base, vp(ts), vp(ti), vp(tc), stream()), "b200ms_topk")
        fs, fi, fc = to_host((ts, ti, tc))
        assert np.array_equal(got[3], fc)
        assert np.array_equal(got[1][:, :, 0], fi)
        assert np.array_equal(bits_of(got[0][:, :, 0]), bits_of(fs))
        assert np.array_equal(got[2], (np.arange(k)[None, :] < fc[:, None]).astype(np.int32))
    h.close()


# ------------------------------------------------------------------------------------------------ 2. full scans
def _unit(rng, n):
    x = rng.standard_normal((n, 128)).astype(np.float32)
    return x / np.maximum(np.linalg.norm(x, axis=1, keepdims=True), 1e-9)


def _docs_corpus(seed, n_docs=40):
    """Documents of 1-40 pages, some pages empty, some pages exact copies (ties across and within documents)."""
    rng = np.random.default_rng(seed)
    pages, page_doc = [], []
    for d in range(n_docs):
        for _ in range(int(rng.integers(1, 41))):
            n = int(rng.choice([0, 1, 5, 31, 33, 70, 130], p=[0.05, 0.15, 0.2, 0.15, 0.15, 0.2, 0.1]))
            pages.append(_unit(rng, n))
            page_doc.append(d)
    for i in rng.choice(len(pages), size=len(pages) // 10, replace=False):
        pages[i] = pages[int(rng.integers(0, len(pages)))].copy()
    page_doc = np.asarray(page_doc, np.int32)
    page_doc[rng.random(len(page_doc)) < 0.03] = -1
    return pages, page_doc, n_docs


PAGES, PAGE_DOC, N_DOCS = _docs_corpus(11)
DTYPES = ["bf16", "int8", "fp8", "binary"]
_INDEXES = {}


def _index(dtype, tier="hbm"):
    key = (dtype, tier)
    if key not in _INDEXES:
        idx = MaxSimIndex(dtype=dtype, tier=tier)
        idx.add_pages(PAGES)
        idx._attach()
        _INDEXES[key] = idx
    return _INDEXES[key]


def _queries(seed, lens=(5, 33, 70)):
    rng = np.random.default_rng(seed)
    qs = [_unit(rng, n) for n in lens]
    qs[0][:3] = PAGES[7][:3] if len(PAGES[7]) >= 3 else qs[0][:3]
    return qs


def _flat_grouped(idx, q_dev, lens, k, per_doc, masks, mask_index, id_base=0):
    """Host grouping of search_device(k = n_pages)'s ranking."""
    n = idx.n_pages
    ts, ti, tc = idx.search_device(q_dev, lens, n, allow_mask_dev=masks, mask_index_dev=mask_index, id_base=id_base)
    ts, ti, tc = to_host((ts, ti, tc))
    return stack_expected([group_flat(ts[q], ti[q], int(tc[q]), PAGE_DOC, N_DOCS, k, per_doc, id_base) for q in range(len(lens))])


@pytest.mark.parametrize("dtype", DTYPES)
def test_search_docs_equals_grouped_flat_ranking(dtype):
    idx = _index(dtype)
    qs = _queries(3)
    lens = [len(q) for q in qs]
    q_dev = torch.from_numpy(np.concatenate(qs)).cuda()
    pd = torch.from_numpy(PAGE_DOC).cuda()
    n = idx.n_pages
    words = (n + 31) // 32
    rng = np.random.default_rng(5)
    m1 = torch.from_numpy(mask_words(rng.random(n) < 0.6).view(np.int32)).cuda()
    mat = torch.from_numpy(np.stack([mask_words(rng.random(n) < p) for p in (0.3, 0.8)]).view(np.int32)).cuda()
    mi = torch.tensor([1, -1, 0], dtype=torch.int32, device="cuda")
    assert mat.shape == (2, words)
    for k, per_doc in [(10, 1), (7, 3), (N_DOCS + 5, 64)]:
        for masks, index in [(None, None), (m1, None), (mat, mi)]:
            got = to_host(idx.search_docs_device(q_dev, lens, k, per_doc, pd, N_DOCS, allow_mask_dev=masks,
                                                 mask_index_dev=index, id_base=1000))
            if masks is not None and index is None:
                index_f, masks_f = torch.zeros(3, dtype=torch.int32, device="cuda"), masks.view(1, -1)
            else:
                index_f, masks_f = index, masks
            want = _flat_grouped(idx, q_dev, lens, k, per_doc, masks_f, index_f, id_base=1000)
            assert_same(got, want, (dtype, k, per_doc, index is not None))
    if dtype in ("int8", "binary"):  # exact integer scores: also the oracle over the raw group scores
        gsc, goff, _, _ = idx.score_groups(qs)
        torch.cuda.synchronize()
        raw = gsc[:, :n].cpu().numpy().astype(np.int64)
        got = to_host(idx.search_docs_device(q_dev, lens, 9, 4, pd, N_DOCS))
        want = []
        for q in range(len(qs)):
            acc = raw[goff[q]:goff[q + 1]].sum(axis=0)
            pos, ids, pc, nd = topk_docs_np(acc, PAGE_DOC, N_DOCS, 9, 4)
            rep = (acc.astype(F32) * F32(idx.score_scale)).astype(F32)
            want.append((np.where(pos >= 0, rep[np.maximum(pos, 0)], F32(-np.inf)).astype(F32), ids, pc, nd))
        assert_same(got, stack_expected(want), dtype)


def test_search_docs_zero_pad_compat():
    idx = MaxSimIndex(dtype="bf16")
    idx.add_pages(PAGES)
    idx.set_option("zero_pad_compat", 128)
    qs = _queries(4)
    lens = [len(q) for q in qs]
    q_dev = torch.from_numpy(np.concatenate(qs)).cuda()
    got = to_host(idx.search_docs_device(q_dev, lens, 12, 3, torch.from_numpy(PAGE_DOC).cuda(), N_DOCS))
    assert_same(got, _flat_grouped(idx, q_dev, lens, 12, 3, None, None), "zero_pad_compat")
    idx.close()


def test_search_docs_above_8192_pages():
    rng = np.random.default_rng(21)
    n = 9000
    pages = [_unit(rng, int(x)) for x in rng.integers(1, 5, size=n)]
    page_doc, n_docs = doc_table(rng, n, "runs")
    idx = MaxSimIndex(dtype="bf16")
    idx.add_pages(pages)
    qs = [_unit(rng, 40), _unit(rng, 3)]
    lens = [len(q) for q in qs]
    q_dev = torch.from_numpy(np.concatenate(qs)).cuda()
    got = to_host(idx.search_docs_device(q_dev, lens, 50, 3, torch.from_numpy(page_doc).cuda(), n_docs))
    gsc, goff, _, _ = idx.score_groups(qs)
    torch.cuda.synchronize()
    raw = gsc[:, :n].cpu().numpy()
    want = []
    for q in range(len(qs)):
        acc = np.zeros(n, F32)
        for g in range(goff[q], goff[q + 1]):
            acc = (acc + raw[g]).astype(F32)
        pos, ids, pc, nd = topk_docs_np(acc, page_doc, n_docs, 50, 3)
        want.append((np.where(pos >= 0, acc[np.maximum(pos, 0)], F32(-np.inf)).astype(F32), ids, pc, nd))
    assert_same(got, stack_expected(want), "9000 pages")
    idx.close()


# ------------------------------------------------------------------------------------------------ 3. candidate lists
def _cand_lists(n_q, n_cand, seed):
    rng = np.random.default_rng(seed)
    n = len(PAGES)
    ids = rng.integers(0, n, size=(n_q, n_cand)).astype(np.int64)
    ids[rng.random(ids.shape) < 0.1] = -1
    ids[rng.random(ids.shape) < 0.05] = n + 5
    for q in range(n_q):  # repeated pages, also of the best candidates
        src = rng.integers(0, n_cand, size=n_cand // 6)
        dst = rng.integers(0, n_cand, size=n_cand // 6)
        ids[q, dst] = ids[q, src]
    return ids


@pytest.mark.parametrize("dtype", DTYPES)
def test_rerank_docs_equals_grouped_rerank(dtype):
    qs = _queries(6, lens=(12, 40, 1, 65))
    lens = [len(q) for q in qs]
    q_dev = torch.from_numpy(np.concatenate(qs)).cuda()
    pd = torch.from_numpy(PAGE_DOC).cuda()
    for n_cand, k, per_doc in [(90, 8, 3), (1500, 20, 2), (37, 64, 64)]:
        cand = torch.from_numpy(_cand_lists(len(qs), n_cand, n_cand)).cuda()
        results = []
        for tier in ("hbm", "host"):
            idx = _index(dtype, tier)
            got = to_host(idx.rerank_docs_batch(q_dev, lens, cand, k, per_doc, pd, N_DOCS))
            ts, ti, tc = to_host(idx.rerank_batch(q_dev, lens, cand, n_cand))
            kk = min(k, n_cand)
            want = stack_expected([group_flat(ts[q], ti[q], int(tc[q]), PAGE_DOC, N_DOCS, kk, per_doc) for q in range(len(qs))])
            assert_same(got, want, (dtype, tier, n_cand))
            results.append(got)
        for a, b in zip(*results):  # host tier == HBM tier, bit for bit
            assert np.array_equal(np.asarray(a).view(np.uint8), np.asarray(b).view(np.uint8))


# ------------------------------------------------------------------------------------------------ 4. refusals
def test_refusals_launch_nothing():
    idx = _index("bf16")
    h = idx.h
    n = idx.n_pages
    q = torch.zeros((4, 128), dtype=torch.float32, device="cuda")
    pd = torch.from_numpy(PAGE_DOC).cuda()
    cand = torch.zeros((1, 8), dtype=torch.int64, device="cuda")
    out = torch.empty(1 << 20, dtype=torch.float32, device="cuda")
    ids = torch.empty(1 << 20, dtype=torch.int64, device="cuda")
    cnt = torch.empty(1 << 16, dtype=torch.int32, device="cuda")
    gs = torch.zeros((4, n + 32), dtype=torch.float32, device="cuda")
    lens = nat.i32_array([4])

    def search(hp=h.ptr, k=5, per_doc=2, pdp=vp(pd), n_docs=N_DOCS, ts=vp(out), ti=vp(ids), pc=vp(cnt), dc=vp(cnt), n_q=1):
        return nat.lib.b200ms_search_docs_device(hp, vp(q), nat.F32, lens, n_q, k, per_doc, pdp, n_docs, None, 0, None,
                                                 ctypes.c_float(1), ctypes.c_float(1), 0, ts, ti, pc, dc, None)

    def rerank(hp=h.ptr, k=5, per_doc=2, pdp=vp(pd), n_docs=N_DOCS, ts=vp(out), ti=vp(ids), pc=vp(cnt), dc=vp(cnt), n_cand=8):
        return nat.lib.b200ms_rerank_docs_batch_device(hp, vp(q), nat.F32, lens, 1, vp(cand), n_cand, k, per_doc, pdp, n_docs,
                                                       ctypes.c_float(1), ctypes.c_float(1), ts, ti, pc, dc, None)

    def topk(hp=h.ptr, k=5, per_doc=2, pdp=vp(pd), n_docs=N_DOCS, ts=vp(out), ti=vp(ids), pc=vp(cnt), dc=vp(cnt), n_pages=n):
        return nat.lib.b200ms_topk_docs(hp, vp(gs), nat.F32, n_pages, n + 32, nat.i32_array([0, 1]), 1, None, pdp, n_docs, k,
                                        per_doc, ctypes.c_float(1), 0, ts, ti, pc, dc, None)

    torch.cuda.synchronize()
    before = nat.lib.b200ms_launch_count(h.ptr)
    for fn in (search, rerank, topk):
        assert fn(hp=None) == EINVAL
        for kw in ({"pdp": None}, {"ts": None}, {"ti": None}, {"pc": None}, {"dc": None}, {"k": 0}, {"k": 4097},
                   {"per_doc": 0}, {"per_doc": 65}, {"n_docs": 0}, {"n_docs": n + 1}, {"n_docs": -1}):
            assert fn(**kw) == EINVAL, (fn.__name__, kw)
    assert search(n_q=0) == EINVAL
    assert rerank(n_cand=0) == EINVAL
    assert topk(n_pages=0, n_docs=1) == EINVAL  # n_docs > n_pages
    assert nat.lib.b200ms_launch_count(h.ptr) == before
    bare = nat.Handle(0)
    assert search(hp=bare.ptr) == ESTATE and rerank(hp=bare.ptr) == ESTATE  # no corpus
    assert nat.lib.b200ms_launch_count(bare.ptr) == 0
    bare.close()
    host = _index("bf16", "host")
    before = nat.lib.b200ms_launch_count(host.h.ptr)
    assert search(hp=host.h.ptr) == ESTATE  # a full scan of a host-resident corpus
    assert nat.lib.b200ms_launch_count(host.h.ptr) == before


# ------------------------------------------------------------------------------------------------ 5. the store
def _run(coro):
    return asyncio.run(coro)


def _store_chunks(seed, n_docs=12):
    rng = np.random.default_rng(seed)
    out = []
    for d in range(n_docs):
        for c in range(int(rng.integers(1, 9))):
            out.append(DocumentChunk(document_id=f"doc{d}", chunk_number=c, content=f"{d}-{c}", metadata={"d": d},
                                     embedding=_unit(rng, int(rng.integers(1, 120)))))
    return out


def _grouped_batch(store, q, k, per, doc_ids=None, app_id=None, min_score=None):
    flat = _run(store.query_similar_batch([q], k=len(store.catalog), doc_ids=doc_ids, app_id=app_id, min_score=min_score))[0]
    order, groups = [], {}
    for c in flat:
        if c.document_id not in groups:
            if len(order) == k:
                continue
            order.append(c.document_id)
            groups[c.document_id] = []
        if len(groups[c.document_id]) < per:
            groups[c.document_id].append(c)
    return [groups[d] for d in order]


def _key(groups):
    return [[(c.document_id, c.chunk_number, np.float32(c.score).view(np.uint32).item(), c.content) for c in g] for g in groups]


@pytest.mark.parametrize("kind", ["exhaustive", "fde", "host"])
def test_store_query_similar_documents(kind):
    kw = {"exhaustive": {}, "fde": {"fde_candidates": 4096}, "host": {"fde_candidates": 4096, "corpus_tier": "host"}}[kind]
    store = B200MultiVectorStore(mode="bf16", compact_dead_fraction=0.2, **kw)
    chunks = _store_chunks(31)
    _run(store.store_embeddings(chunks))
    rng = np.random.default_rng(32)
    q = _unit(rng, 20)
    q[:2] = chunks[3].embedding[:2]

    def check(k, per, **f):
        got = _run(store.query_similar_documents(q, k, pages_per_document=per, **f))
        assert _key(got) == _key(_grouped_batch(store, q, k, per, **f)), (kind, k, per, f)
        return got

    check(3, 1)
    check(5, 4)
    assert len(check(100, 64)) == 12
    check(4, 2, doc_ids=["doc1", "doc5", "doc9", "nope"])
    got = check(10, 3, min_score=float(np.median([c.score for g in check(12, 8) for c in g])))
    assert all(g for g in got)
    assert _run(store.query_similar_documents(q, 5, doc_ids=[])) == []
    n_before = len(store.catalog)
    for d in ("doc0", "doc2", "doc3", "doc4"):  # crosses compact_dead_fraction: the corpus and the ordinals are rebuilt
        assert _run(store.delete_chunks_by_document_id(d))
    assert len(store.catalog) < n_before  # compacted
    got = check(6, 3)
    assert not {"doc0", "doc2", "doc3", "doc4"} & {g[0].document_id for g in got}
    store.close()
