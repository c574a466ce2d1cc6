"""Documents ranked by document-level MaxSim on an H100 (run with -m gpu): b200ms_search_doc_maxsim_device,
b200ms_rerank_doc_maxsim_batch_device, MaxSimIndex / TwoStageSearch.search_doc_maxsim and the store's
query_similar_documents(score_by="document").

Every corpus dtype, against tests/doc_maxsim_oracle.py on the oracle's own rounding of the same inputs (int8 and 1-bit
exact to the bit, bf16 and fp8 within the float tolerances of test_gpu_parity.py), on a corpus with one-page documents, a
document larger than one work unit, documents whose pages are interleaved with other documents' pages, deleted pages (a
page_doc of -1), an empty page and a document without pages; queries of 1, 32 and 1030 tokens and a mixed batch with
per-query masks; the FDE and sign first stages; crafted candidate lists; the value cases of test_gpu_scorer_values.py
(inf, NaN, signed zeros) and the int32 limits of test_gpu_integer_limits.py; a corpus past 4 GiB; a batch whose token
table passes the 1 GiB bound (several passes) and a query that alone passes it (refused); the host tier (refused).
A one-page document scores bit for bit its search_device page score throughout.
"""
import asyncio
import gc

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

torch = pytest.importorskip("torch")
if not torch.cuda.is_available():  # pragma: no cover - the gpu marker normally deselects these on CPU boxes
    pytest.skip("CUDA device required", allow_module_level=True)

import scale_reference as sr  # noqa: E402
from doc_maxsim_oracle import doc_maxsim_np, finish  # noqa: E402
from explain_oracle import maxsim_explain_np, quantise  # noqa: E402
from mmr_oracle import quantise_rows  # noqa: E402
from morphik_core_b200 import _native as nat  # noqa: E402
from morphik_core_b200.fde import TwoStageIndex  # noqa: E402
from morphik_core_b200.index import MaxSimIndex  # noqa: E402
from morphik_core_b200.models import DocumentChunk  # noqa: E402
from morphik_core_b200.signs import SignTwoStageIndex  # noqa: E402
from morphik_core_b200.store import DOCUMENT_SCORE_KEY, B200MultiVectorStore  # noqa: E402

DEV = torch.device("cuda", 0)
KIND = {"bf16": "bf16", "int8": "int8", "fp8": "fp8", "binary": "bits"}
DTYPES = list(KIND)
EXACT = ("int8", "binary")
RTOL = 1e-3  # test_gpu_parity.BF16_RTOL

# ------------------------------------------------------------------------------------------------ the corpus
N_SINGLE = 30           # pages 0..29: one document each
BIG = range(30, 38)     # document 30: 8 pages of 700 rows, more than one 4096-row work unit
N_DOCS = 41             # documents 31..39: the pages from 38 on, interleaved; document 40 has no page


def _unit(rng, n):
    x = rng.standard_normal((n, 128)).astype(np.float32)
    return x / np.maximum(np.linalg.norm(x, axis=1, keepdims=True), 1e-9)


def _layout(seed=3, n_pages=200):
    rng = np.random.default_rng(seed)
    lens = rng.integers(1, 65, n_pages)
    lens[list(BIG)] = 700
    lens[n_pages - 1] = 0  # an empty page of document 31 + (199 % 9)
    pages = [_unit(rng, int(n)) for n in lens]
    page_doc = np.empty(n_pages, np.int32)
    page_doc[:N_SINGLE] = np.arange(N_SINGLE)
    page_doc[list(BIG)] = 30
    rest = np.arange(BIG.stop, n_pages)
    page_doc[rest] = 31 + rest % 9
    page_doc[rest[rest % 13 == 0]] = -1  # deleted pages
    return pages, page_doc


PAGES, PAGE_DOC = _layout()
N_PAGES = len(PAGES)
LENS = np.array([len(p) for p in PAGES])
OFF = np.concatenate([[0], np.cumsum(LENS)])
_ROWS = {}


def quantised_rows(dtype):
    if dtype not in _ROWS:
        _ROWS[dtype] = quantise(np.concatenate(PAGES), KIND[dtype])
    return _ROWS[dtype]


def queries(lens, seed):
    """Unit tokens; every other token is a row of some page, so tokens have clear best pages in several documents."""
    rng = np.random.default_rng(seed)
    all_rows = np.concatenate(PAGES)
    out = []
    for n in lens:
        q = _unit(rng, n)
        pick = rng.integers(0, len(all_rows), n)
        q[::2] = 0.7 * all_rows[pick[::2]] + 0.3 * q[::2]
        out.append(q)
    return out


def token_maxima(dtype, q):
    """m [n_pages, T] on the oracle's rounding (raw units: int8 / 1-bit exact integers)."""
    best, _, _ = maxsim_explain_np(quantise(q, KIND[dtype]), quantised_rows(dtype), OFF, KIND[dtype])
    return best


def words_of(allow):
    b = np.packbits(np.asarray(allow, bool), bitorder="little")
    b = np.concatenate([b, np.zeros((-len(b)) % 4, np.uint8)])
    return b.view(np.uint32)


APP_PAGES = (np.arange(N_PAGES) % 3) != 1  # an app_id filter: the pages stored under the caller's app
FILTERS = {"none": None, "doc_ids": np.isin(PAGE_DOC, [2, 5, 30, 31, 33, 36, 40]), "app_id": APP_PAGES}


def reported(dtype, idx, raw):
    """What the device reports for a raw sum: exact kinds fp32(fp32(finish(S)) * scale)."""
    if dtype in EXACT:
        return np.float32(np.float32(finish(raw, True)) * np.float32(idx.score_scale))
    return raw * idx.score_scale


def check_query(dtype, idx, q, got, k, per_doc, allow=None, docs_allowed=None, what=""):
    """got = (doc scores [k], doc ids [k], evidence ids [k, per_doc], shares [k, per_doc], counts [k], found) of one query."""
    ds, di, ei, es, ec, dc = got
    counted = LENS > 0
    if allow is not None:
        counted &= np.asarray(allow, bool)
    if docs_allowed is not None:
        counted &= np.isin(PAGE_DOC, list(docs_allowed))
    m = token_maxima(dtype, q)
    docs, S, ev = doc_maxsim_np(m, PAGE_DOC, N_DOCS, k, per_doc, counted)
    n = len(docs)
    assert int(dc) == n, (what, dc, n)
    assert (di[n:] == -1).all() and np.isneginf(ds[n:]).all() and (ec[n:] == 0).all(), what
    assert (ei[n:] == -1).all() and np.isneginf(es[n:]).all(), what
    if dtype in EXACT:
        assert di[:n].tolist() == docs.tolist(), what
        assert ds[:n].view(np.uint32).tolist() == np.array([reported(dtype, idx, s) for s in S], np.float32).view(np.uint32).tolist(), what
        for i, (pages, shares) in enumerate(ev):
            assert ec[i] == len(pages) and ei[i, :len(pages)].tolist() == pages.tolist(), (what, i)
            want = np.array([reported(dtype, idx, s) for s in shares], np.float32)
            assert es[i, :len(pages)].view(np.uint32).tolist() == want.view(np.uint32).tolist(), (what, i)
            assert np.isneginf(es[i, len(pages):]).all() and (ei[i, len(pages):] == -1).all()
        return
    # floats: every returned document's score and the ranked score list match within rounding; evidence pages belong to
    # the document, carry their oracle shares and are ordered
    Sd = dict(zip(docs.tolist(), S.tolist()))
    all_S = doc_maxsim_np(m, PAGE_DOC, N_DOCS, N_DOCS, 1, counted)
    Sall = dict(zip(all_S[0].tolist(), all_S[1].tolist()))
    scale = idx.score_scale
    tol = lambda v: RTOL * abs(v) + 1e-4 * scale * q.shape[0]  # noqa: E731
    for i in range(n):
        d = int(di[i])
        assert d in Sall and abs(ds[i] - Sall[d] * scale) <= tol(Sall[d] * scale), (what, i, d, ds[i], Sall.get(d))
        assert abs(ds[i] - Sd[int(docs[i])] * scale) <= tol(ds[i]), (what, i)
        pages = ei[i, :ec[i]]
        assert ec[i] >= 1 and (PAGE_DOC[pages] == d).all() and counted[pages].all(), (what, i)
        assert len(set(pages.tolist())) == len(pages)
        assert all(a >= b - tol(a) for a, b in zip(es[i, :ec[i]], es[i, 1:ec[i]])), (what, i)
        if ec[i] < per_doc:  # every evidence page is listed: the shares add up to the score
            assert abs(es[i, :ec[i]].astype(np.float64).sum() - ds[i]) <= tol(ds[i]), (what, i)
    assert np.all(np.diff(ds[:n]) <= 1e-6 * np.abs(ds[:n]).max(initial=1.0)), what


def check_single_pages(idx, qs, got_batch, allow=None):
    """A one-page document's score is the bits of its page's search_device score."""
    src = torch.from_numpy(np.concatenate(qs)).to(DEV)
    lens = [len(q) for q in qs]
    mask = None if allow is None else torch.from_numpy(words_of(allow).view(np.int32)).to(DEV)
    ts, ti, tc = idx.search_device(src, lens, N_PAGES, allow_mask_dev=mask)
    ts, ti = ts.cpu().numpy(), ti.cpu().numpy()
    seen = 0
    for qi in range(len(qs)):
        page_score = {int(p): s for p, s in zip(ti[qi], ts[qi]) if p >= 0}
        ds, di = got_batch[0][qi], got_batch[1][qi]
        for s, d in zip(ds, di):
            if 0 <= d < N_SINGLE:
                assert np.float32(s).view(np.uint32) == np.float32(page_score[int(d)]).view(np.uint32), (qi, d)
                seen += 1
    return seen


_IDX = {}


def index(dtype):
    if dtype not in _IDX:
        idx = MaxSimIndex(dtype=dtype)
        idx.add_pages(PAGES)
        _IDX[dtype] = idx
    return _IDX[dtype]


def page_doc_dev(n=None):
    return torch.from_numpy(PAGE_DOC if n is None else n).to(DEV)


def run_device(idx, qs, k, per_doc, allow=None, mask_rows=None, mask_index=None):
    src = torch.from_numpy(np.concatenate(qs)).to(DEV)
    if mask_rows is not None:
        masks = torch.from_numpy(np.stack([words_of(a) for a in mask_rows]).view(np.int32)).to(DEV)
        mi = torch.tensor(mask_index, dtype=torch.int32, device=DEV)
    else:
        masks = None if allow is None else torch.from_numpy(words_of(allow).view(np.int32)).to(DEV)
        mi = None
    out = idx.search_doc_maxsim_device(src, [len(q) for q in qs], k, per_doc, page_doc_dev(), N_DOCS, masks, mi)
    return tuple(t.cpu().numpy() for t in out)


# ------------------------------------------------------------------------------------------------ exhaustive
@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("filt", list(FILTERS))
@pytest.mark.parametrize("qlens", [[1], [32], [1030]], ids=["q1", "q32", "q1030"])
def test_search_matches_the_oracle(dtype, filt, qlens):
    idx = index(dtype)
    qs = queries(qlens, seed=len(qlens) + qlens[0])
    allow = FILTERS[filt]
    k, per_doc = 12, 5
    got = run_device(idx, qs, k, per_doc, allow=allow)
    check_query(dtype, idx, qs[0], tuple(x[0] for x in got), k, per_doc, allow, what=(dtype, filt, qlens))
    host = idx.search_doc_maxsim(qs, k, per_doc, page_doc_dev(), N_DOCS,
                                 allow_mask=None if allow is None else words_of(allow))
    for a, b in zip(host, got):
        assert np.array_equal(np.asarray(a).view(np.uint8), np.asarray(b).view(np.uint8))
    got_all = run_device(idx, qs, N_DOCS, 1, allow=allow)
    assert check_single_pages(idx, qs, got_all, allow) > 0


@pytest.mark.parametrize("dtype", DTYPES)
def test_mixed_batch_with_per_query_masks(dtype):
    idx = index(dtype)
    qlens = [1, 32, 1030, 7, 65, 33]
    qs = queries(qlens, seed=11)
    rows = [FILTERS["doc_ids"], APP_PAGES, np.arange(N_PAGES) >= 30]
    mi = [0, -1, 1, 2, 0, -1]
    k, per_doc = 8, 3
    got = run_device(idx, qs, k, per_doc, mask_rows=rows, mask_index=mi)
    for i, q in enumerate(qs):
        allow = None if mi[i] < 0 else rows[mi[i]]
        check_query(dtype, idx, q, tuple(x[i] for x in got), k, per_doc, allow, what=(dtype, i))
    # each query alone gives the same bits as in the batch
    for i in (0, 2, 3):
        one = run_device(idx, [qs[i]], k, per_doc, allow=None if mi[i] < 0 else rows[mi[i]])
        for a, b in zip(one, got):
            assert np.array_equal(np.atleast_1d(a[0]).view(np.uint8), np.atleast_1d(b[i]).view(np.uint8)), (dtype, i)


# ------------------------------------------------------------------------------------------------ two stages
def _first_stage(stage, dtype):
    if stage == "fde":
        two = TwoStageIndex(dtype=dtype)
    else:
        if dtype == "binary":
            pytest.skip("the sign first stage needs a corpus with more precise rows than its signs")
        two = SignTwoStageIndex(dtype=dtype)
    two.add_pages(PAGES)
    return two


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("stage", ["fde", "sign"])
@pytest.mark.parametrize("filt", list(FILTERS))
def test_two_stage_scores_the_candidates_documents(dtype, stage, filt):
    two = _first_stage(stage, dtype)
    try:
        qs = queries([32, 1030], seed=23)
        allow = FILTERS[filt]
        words = None if allow is None else words_of(allow)
        k, per_doc, n_cand = 6, 4, 20
        got = two.search_doc_maxsim(qs, k, per_doc, page_doc_dev(), N_DOCS, n_candidates=n_cand, allow_mask=words)
        mask_dev = None if words is None else torch.from_numpy(words.view(np.int32)).to(DEV)
        ci, _, tc = two.candidates(qs, n_cand, mask_dev)
        ci = ci.cpu().numpy()
        for i, q in enumerate(qs):
            c = ci[i][ci[i] >= 0]
            assert len(c) > 0
            cand_docs = {int(d) for d in PAGE_DOC[c] if d >= 0}
            check_query(dtype, two.index, q, tuple(x[i] for x in got), k, per_doc, allow, cand_docs, (dtype, stage, filt, i))
        # every page a candidate: the exhaustive result
        full = two.search_doc_maxsim(qs, k, per_doc, page_doc_dev(), N_DOCS, n_candidates=N_PAGES, allow_mask=words)
        want = run_device(two.index, qs, k, per_doc, allow=allow)
        for a, b in zip(full, want):
            assert np.array_equal(np.asarray(a).view(np.uint8), np.asarray(b).view(np.uint8))
    finally:
        two.index.close()


@pytest.mark.parametrize("dtype", DTYPES)
def test_rerank_batch_over_crafted_candidate_lists(dtype):
    idx = index(dtype)
    qs = queries([32, 5, 1030], seed=31)
    lists = np.array([[3, -1, 45, 45, N_PAGES + 7, 39],      # a single-page document, interleaved documents, repeats
                      [-1, -1, -1, -1, -1, -1],              # nothing: no document
                      [31, 26, 52, 13 * 4, 199, 0]], np.int64)  # the big document, a deleted page, the empty page
    cand = torch.from_numpy(lists).to(DEV)
    src = torch.from_numpy(np.concatenate(qs)).to(DEV)
    allow = APP_PAGES
    mask = torch.from_numpy(words_of(allow).view(np.int32)).to(DEV)
    for m in (None, mask):
        out = idx.rerank_doc_maxsim_batch(src, [len(q) for q in qs], cand, 9, 3, page_doc_dev(), N_DOCS, allow_mask_dev=m,
                                          id_base=1000)
        got = [t.cpu().numpy() for t in out]
        got[2] = np.where(got[2] >= 0, got[2] - 1000, -1)
        for i, q in enumerate(qs):
            c = lists[i][(lists[i] >= 0) & (lists[i] < N_PAGES)]
            docs = {int(d) for d in PAGE_DOC[c] if d >= 0}
            check_query(dtype, idx, q, tuple(x[i] for x in got), 9, 3, None if m is None else allow, docs, (dtype, i))
    assert got[5][1] == 0


# ------------------------------------------------------------------------------------------------ values and limits
def _value_index(dtype, rows_per_page):
    idx = MaxSimIndex(dtype=dtype)
    idx.add_pages(rows_per_page)
    return idx


@pytest.mark.parametrize("dtype", ["bf16", "fp8"])
def test_inf_nan_and_signed_zero_tokens(dtype):
    """Rows with one nonzero element: every product is exact, so token maxima and sums are exact floats, NaN included."""
    specials = [1.0, 2.0, -3.0, np.inf, -np.inf, np.nan, 0.0, -0.0, 0.5]
    rng = np.random.default_rng(5)
    pages, owners = [], []
    for p in range(24):
        n = int(rng.integers(1, 5))
        rows = np.zeros((n, 128), np.float32)
        for r in range(n):
            rows[r, int(rng.integers(0, 4))] = specials[int(rng.integers(0, len(specials)))] / (64.0 if dtype == "fp8" else 1.0)
        pages.append(rows)
        owners.append(p if p < 6 else 6 + p % 5)
    page_doc = np.array(owners, np.int32)
    idx = _value_index(dtype, pages)
    try:
        scale = 1.0 / 64.0 if dtype == "fp8" else 1.0
        tokens = np.zeros((9, 128), np.float32)
        for t in range(9):
            tokens[t, t % 4] = [1.0, -1.0, 0.0, 2.0][t % 4] * scale
        q = tokens
        src = torch.from_numpy(q).to(DEV)
        n_docs = 11
        out = idx.search_doc_maxsim_device(src, [len(q)], n_docs, 4, torch.from_numpy(page_doc).to(DEV), n_docs)
        ds, di, ei, es, ec, dc = (t.cpu().numpy()[0] for t in out)
        lens = np.array([len(p) for p in pages])
        off = np.concatenate([[0], np.cumsum(lens)])
        # products one by one (a BLAS matmul does not keep IEEE non-finite arithmetic: 0 * inf leaks into other entries)
        qq, rr = quantise_rows(q, KIND[dtype]).astype(np.float64), quantise_rows(np.concatenate(pages), KIND[dtype]).astype(np.float64)
        with np.errstate(invalid="ignore"):
            sim = (qq[:, None, :] * rr[None, :, :]).sum(axis=2)  # [T, rows]
            m = np.stack([np.fmax.reduce(sim[:, off[p]:off[p + 1]], axis=1) for p in range(len(pages))])
        docs, S, ev = doc_maxsim_np(m, page_doc, n_docs, n_docs, 4)
        assert int(dc) == len(docs)
        want = np.array([s * idx.score_scale for s in S], np.float32)
        got_by_doc = dict(zip(di[:dc].tolist(), ds[:dc].tolist()))
        for d, w in zip(docs.tolist(), want):
            g = np.float32(got_by_doc[d])
            assert (np.isnan(g) and np.isnan(w)) or g.view(np.uint32) == np.float32(w).view(np.uint32), (d, g, w)
        # the NaN ranks first, then numbers in order, ties to the lower ordinal: the oracle's order
        assert di[:dc].tolist() == docs.tolist()
        ts, ti, tc = idx.search_device(src, [len(q)], len(pages))
        page_score = dict(zip(ti[0].cpu().numpy().tolist(), ts[0].cpu().numpy().tolist()))
        for s, d in zip(ds[:dc], di[:dc]):
            if d < 6:
                assert np.float32(s).view(np.uint32) == np.float32(page_score[int(d)]).view(np.uint32) or (
                    np.isnan(s) and np.isnan(page_score[int(d)]))
    finally:
        idx.close()


@pytest.mark.parametrize("dtype", EXACT)
def test_integer_sums_saturate_like_page_scores(dtype):
    """1041 tokens at the integer limit: S passes 2^31 and reports the bound, as the page scores do."""
    rng = np.random.default_rng(9)
    base = -np.ones((1, 128), np.float32) * 2.0
    pages = [np.repeat(base, n, axis=0) for n in (3, 40, 1, 2)] + [_unit(rng, 5)]
    page_doc = np.array([0, 1, 1, 2, 2], np.int32)
    idx = _value_index(dtype, pages)
    try:
        q = np.repeat(base, 1041, axis=0)
        src = torch.from_numpy(q).to(DEV)
        out = idx.search_doc_maxsim_device(src, [1041], 3, 2, torch.from_numpy(page_doc).to(DEV), 3)
        ds, di, ei, es, ec, dc = (t.cpu().numpy()[0] for t in out)
        lens = np.array([len(p) for p in pages])
        off = np.concatenate([[0], np.cumsum(lens)])
        m, _, _ = maxsim_explain_np(quantise(q, KIND[dtype]), quantise(np.concatenate(pages), KIND[dtype]), off, KIND[dtype])
        docs, S, ev = doc_maxsim_np(m, page_doc, 3, 3, 2)
        assert di.tolist() == docs.tolist() and int(dc) == 3
        assert ds.view(np.uint32).tolist() == np.array([reported(dtype, idx, s) for s in S], np.float32).view(np.uint32).tolist()
        if dtype == "int8":
            assert (S == 2**31 - 1).sum() >= 2  # the limit is reached
        ts, ti, tc = idx.search_device(src, [1041], 5)
        page_score = dict(zip(ti[0].cpu().numpy().tolist(), ts[0].cpu().numpy().tolist()))
        assert np.float32(ds[di.tolist().index(0)]).view(np.uint32) == np.float32(page_score[0]).view(np.uint32)
        for i, (pages_, shares) in enumerate(ev):
            assert ei[i, :ec[i]].tolist() == pages_.tolist()
            assert es[i, :ec[i]].view(np.uint32).tolist() == np.array([reported(dtype, idx, s) for s in shares],
                                                                       np.float32).view(np.uint32).tolist()
    finally:
        idx.close()


# ------------------------------------------------------------------------------------------------ sizes
def test_batches_past_the_table_bound_run_in_passes_and_a_single_query_over_it_is_refused():
    """200 000 one-row pages, one document each: a 32-token query needs a 51 MB token table, 24 of them 1.2 GB (two passes),
    a 1030-token query 1.7 GB (refused)."""
    n = 200_000
    rng = np.random.default_rng(2)
    rows = quantise(rng.standard_normal((n, 128)).astype(np.float32) * 0.5, "int8").astype(np.float32) / 127.0
    idx = MaxSimIndex(dtype="int8")
    try:
        idx.add_pages([rows[i:i + 1] for i in range(n)])
        page_doc = torch.arange(n, dtype=torch.int32, device=DEV)
        qs = [(_unit(rng, 32) * 1.0).astype(np.float32) for _ in range(24)]
        src = torch.from_numpy(np.concatenate(qs)).to(DEV)
        batch = [t.cpu().numpy() for t in idx.search_doc_maxsim_device(src, [32] * 24, 10, 1, page_doc, n)]
        for i in (0, 11, 12, 23):
            one = [t.cpu().numpy() for t in idx.search_doc_maxsim_device(src[32 * i:32 * i + 32], [32], 10, 1, page_doc, n)]
            for a, b in zip(one, batch):
                assert np.array_equal(np.atleast_1d(a[0]).view(np.uint8), np.atleast_1d(b[i]).view(np.uint8)), i
        # one-page documents: the page ranking of search_device, bit for bit
        ts, ti, tc = (t.cpu().numpy() for t in idx.search_device(src, [32] * 24, 10))
        assert np.array_equal(batch[1], ti) and np.array_equal(batch[0].view(np.uint32), ts.view(np.uint32))
        long_q = torch.from_numpy(_unit(rng, 1030)).to(DEV)
        with pytest.raises(nat.NativeError, match="token table"):
            idx.search_doc_maxsim_device(long_q, [1030], 10, 1, page_doc, n)
    finally:
        idx.close()
        gc.collect()
        torch.cuda.empty_cache()


def _page_token_maxima(rows_u8, lens, q):
    """float64 [n_pages, T]: the max over each page's true rows of the int8 products (exact)."""
    pad = sr.padded_rows(lens)
    start = np.concatenate([[0], np.cumsum(pad)])
    T = q.shape[0]
    out = torch.zeros((len(lens), T), dtype=torch.float64, device=DEV)
    p0 = 0
    while p0 < len(lens):
        p1 = min(int(np.searchsorted(start, start[p0] + (1 << 20), side="right")) - 1, len(lens))
        p1 = max(p1, p0 + 1)
        r0, r1 = int(start[p0]), int(start[p1])
        if r1 > r0:
            sim = q @ sr.decode("int8", rows_u8[r0:r1]).T
            col = np.arange(r1 - r0) + r0
            page_of_row = np.repeat(np.arange(p0, p1), pad[p0:p1])
            is_pad = torch.from_numpy(col - start[page_of_row] >= lens[page_of_row]).to(DEV)
            sim.masked_fill_(is_pad[None, :], float("-inf"))
            cm = sim.view(T, -1, 32).amax(dim=2)
            cp = torch.from_numpy(page_of_row[::32] - p0).to(DEV)
            best = torch.full((T, p1 - p0), float("-inf"), dtype=torch.float64, device=DEV)
            best.scatter_reduce_(1, cp[None, :].expand(T, -1), cm, "amax", include_self=True)
            out[p0:p1] = best.T
        p0 = p1
    return out.cpu().numpy()


def test_past_4gib_against_the_oracle():
    """The int8 planted corpus of test_gpu_page_query_scale.py (past 4 GiB), documents of 16 consecutive pages except
    that every fifth page belongs to the document after next (interleaved); scores and evidence exact."""
    n_pages = 40960
    rows_needed = int(sr.padded_rows(sr.page_lens(n_pages, 0)).sum())
    gc.collect()
    torch.cuda.empty_cache()
    free, _ = torch.cuda.mem_get_info(DEV)
    if free < rows_needed * 128 + (10 << 30):
        pytest.skip("not enough device memory for the corpus past 4 GiB")
    idx = sr.build("int8", n_pages, 0)
    try:
        assert idx.n_rows_padded * 128 > (1 << 32) + (1 << 30)
        lens = np.asarray(idx.page_lens, np.int64)
        p = np.arange(n_pages)
        page_doc = (p // 16 + np.where(p % 5 == 0, 2, 0)) % (n_pages // 16)
        page_doc = page_doc.astype(np.int32)
        n_docs = n_pages // 16
        qs = sr.queries("int8", 0, [32, 100])
        out = idx.search_doc_maxsim(qs, 10, 4, torch.from_numpy(page_doc).to(DEV), n_docs)
        rows = idx.packed_rows()
        for i, q in enumerate(qs):
            qd = torch.from_numpy(quantise(q, "int8").astype(np.float64)).to(DEV)
            m = np.rint(np.where(lens[:, None] > 0, _page_token_maxima(rows, lens, qd), 0)).astype(np.int64)
            docs, S, ev = doc_maxsim_np(m, page_doc, n_docs, 10, 4, lens > 0)
            ds, di, ei, es, ec, dc = (x[i] for x in out)
            assert di.tolist() == docs.tolist()
            assert ds.view(np.uint32).tolist() == np.array([reported("int8", idx, s) for s in S], np.float32).view(np.uint32).tolist()
            for j, (pg, sh) in enumerate(ev):
                assert ei[j, :ec[j]].tolist() == pg.tolist()
    finally:
        idx.close()
        gc.collect()
        torch.cuda.empty_cache()


# ------------------------------------------------------------------------------------------------ refusals and the store
def test_host_tier_is_refused():
    idx = MaxSimIndex(dtype="bf16", tier="host")
    try:
        idx.add_pages(PAGES[:4])
        q = torch.from_numpy(queries([4], 1)[0]).to(DEV)
        with pytest.raises(ValueError, match="HBM"):
            idx.search_doc_maxsim_device(q, [4], 2, 1, torch.zeros(4, dtype=torch.int32, device=DEV), 1)
        with pytest.raises(ValueError, match="HBM"):
            idx.rerank_doc_maxsim_batch(q, [4], torch.zeros((1, 2), dtype=torch.int64, device=DEV), 2, 1,
                                        torch.zeros(4, dtype=torch.int32, device=DEV), 1)
    finally:
        idx.close()


@pytest.mark.parametrize("stage", ["exhaustive", "fde", "sign"])
def test_store_ranks_documents_as_one_bag(stage):
    kw = {"fde": {"fde_candidates": 400}, "sign": {"sign_candidates": 400}}.get(stage, {})
    store = B200MultiVectorStore(mode="int8", coalesce_queries=False, **kw)
    try:
        chunks = [DocumentChunk(document_id=f"doc{int(PAGE_DOC[p])}" if PAGE_DOC[p] >= 0 else f"gone{p}", chunk_number=p,
                                content=str(p), embedding=PAGES[p], metadata={}) for p in range(N_PAGES) if LENS[p] > 0]
        asyncio.run(store.store_embeddings(chunks))
        for p in range(N_PAGES):
            if PAGE_DOC[p] < 0:
                asyncio.run(store.delete_chunks_by_document_id(f"gone{p}"))
        q = queries([32], 41)[0]
        res = asyncio.run(store.query_similar_documents(q, 5, pages_per_document=3, score_by="document",
                                                        doc_ids=[f"doc{d}" for d in (2, 30, 31, 35)]))
        idx = store._index
        m = token_maxima("int8", q)
        docs, S, ev = doc_maxsim_np(m, PAGE_DOC, N_DOCS, 5, 3, (LENS > 0) & np.isin(PAGE_DOC, [2, 30, 31, 35]))
        assert [lst[0].document_id for lst in res] == [f"doc{d}" for d in docs]
        for lst, s, (pg, sh) in zip(res, S, ev):
            assert [c.chunk_number for c in lst] == pg.tolist()
            assert all(c.metadata[DOCUMENT_SCORE_KEY] == float(reported("int8", idx, s)) for c in lst)
            assert [c.score for c in lst] == [float(reported("int8", idx, x)) for x in sh]
    finally:
        store.close()


@pytest.mark.parametrize("dtype", ["bf16", "binary"])
def test_calls_on_other_streams_wait_for_the_handle(dtype):
    """A document call left in flight on one stream and a search issued right after it on another (and the reverse) both
    return what they return alone: they share the handle's scratch, so the handle orders them."""
    idx = index(dtype)
    qs = queries([1030, 32], seed=51)
    src = torch.from_numpy(np.concatenate(qs)).to(DEV)
    lens = [len(q) for q in qs]
    pd = page_doc_dev()

    def doc_call():
        return idx.search_doc_maxsim_device(src, lens, 10, 4, pd, N_DOCS)

    def page_call():
        return idx.search_device(src, lens, 50)

    alone_doc = [t.cpu().numpy() for t in doc_call()]
    alone_page = [t.cpu().numpy() for t in page_call()]
    s1, s2 = torch.cuda.Stream(DEV), torch.cuda.Stream(DEV)
    for first, second in ((doc_call, page_call), (page_call, doc_call)):
        torch.cuda.synchronize(DEV)
        with torch.cuda.stream(s1):
            a = first()
        with torch.cuda.stream(s2):
            b = second()
        torch.cuda.synchronize(DEV)
        got_doc, got_page = (a, b) if first is doc_call else (b, a)
        for x, y in zip(got_doc, alone_doc):
            assert np.array_equal(x.cpu().numpy().view(np.uint8), y.view(np.uint8))
        for x, y in zip(got_page, alone_page):
            assert np.array_equal(x.cpu().numpy().view(np.uint8), y.view(np.uint8))
