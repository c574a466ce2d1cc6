"""The document-level MaxSim oracle (doc_maxsim_oracle.py) against brute force: a document's rows pooled into one bag and
scored as one page, on every kind, with NaN / inf tokens, arg-max ties, masks, and one-page documents."""
import numpy as np
import pytest

from doc_maxsim_oracle import I32_BOUND, doc_maxsim_np, doc_token_max
from explain_oracle import KINDS, maxsim_explain_np, quantise, similarity_np


def _corpus(kind, seed, n_pages=12, n_docs=4, T=7):
    rng = np.random.default_rng(seed)
    lens = rng.integers(1, 6, n_pages)
    off = np.concatenate([[0], np.cumsum(lens)])
    rows = quantise(rng.standard_normal((off[-1], 128)).astype(np.float32), kind)
    q = quantise(rng.standard_normal((T, 128)).astype(np.float32), kind)
    page_doc = rng.integers(0, n_docs, n_pages)
    return q, rows, off, page_doc


def _brute(q, rows, off, page_doc, d, kind, counted=None):
    """S of document d: its counted pages' rows as one bag, MaxSim of the bag."""
    pages = [p for p in range(len(off) - 1) if page_doc[p] == d and (counted is None or counted[p])]
    bag = np.concatenate([rows[off[p]:off[p + 1]] for p in pages])
    sim = similarity_np(q, bag, kind)
    if kind in ("int8", "bits"):
        return int(sim.max(axis=1).sum())
    return float(np.fmax.reduce(sim, axis=1).sum())


@pytest.mark.parametrize("kind", KINDS)
@pytest.mark.parametrize("seed", [0, 1, 2])
def test_scores_are_maxsim_of_the_pooled_document(kind, seed):
    q, rows, off, page_doc = _corpus(kind, seed)
    m, _, _ = maxsim_explain_np(q, rows, off, kind)
    counted = np.random.default_rng(seed + 9).random(len(page_doc)) < 0.8
    docs, S, ev = doc_maxsim_np(m, page_doc, 4, k=4, per_doc=64, counted=counted)
    want = {d: _brute(q, rows, off, page_doc, d, kind, counted) for d in set(page_doc[counted].tolist())}
    assert sorted(docs.tolist()) == sorted(want)
    for d, s, (pages, shares) in zip(docs, S, ev):
        assert s == pytest.approx(want[int(d)], rel=1e-12)
        assert set(page_doc[pages].tolist()) == {int(d)} and counted[pages].all()
        assert shares.sum() == pytest.approx(s, rel=1e-12)
    assert all(a >= b for a, b in zip(S, S[1:]))


@pytest.mark.parametrize("kind", KINDS)
def test_a_one_page_document_scores_its_page(kind):
    q, rows, off, page_doc = _corpus(kind, 5, n_pages=6, n_docs=6)
    page_doc = np.arange(6)
    m, _, _ = maxsim_explain_np(q, rows, off, kind)
    docs, S, ev = doc_maxsim_np(m, page_doc, 6, k=6, per_doc=2)
    for d, s, (pages, shares) in zip(docs, S, ev):
        assert s == m[d].sum() and pages.tolist() == [d] and shares.tolist() == [s]


def test_ties_go_to_the_lower_page_and_the_lower_document():
    m = np.array([[1.0, 2.0], [1.0, 3.0], [1.0, 3.0], [4.0, 1.0]])
    M, B, found = doc_token_max(m, [0, 0, 0, 1], 2)
    assert B.tolist() == [[0, 1], [3, 3]] and M.tolist() == [[1.0, 3.0], [4.0, 1.0]]
    docs, S, ev = doc_maxsim_np(m, [0, 0, 0, 1], 2, k=2, per_doc=4)
    assert docs.tolist() == [1, 0] and S.tolist() == [5.0, 4.0] and ev[1][0].tolist() == [1, 0]
    docs, S, ev = doc_maxsim_np(m, [0, 1, 1, 2], 3, k=3, per_doc=4)
    assert docs.tolist() == [2, 1, 0]  # 5, 4 and 3
    docs, S, _ = doc_maxsim_np(np.array([[2.0], [2.0]]), [1, 0], 2, k=2, per_doc=1)
    assert docs.tolist() == [0, 1]  # tied scores: the lower ordinal first
    # evidence: equal shares go to the lower page
    _, _, ev = doc_maxsim_np(np.array([[5.0, 0.0], [0.0, 5.0]]), [0, 0], 1, k=1, per_doc=2)
    assert ev[0][0].tolist() == [0, 1]


def test_nan_loses_to_any_number_and_signed_zeros_rank():
    nan, inf = np.nan, np.inf
    m = np.array([[nan, nan, -0.0, 1.0], [-inf, nan, 0.0, inf], [nan, nan, -0.0, -1.0]])
    M, B, _ = doc_token_max(m, [0, 0, 0], 1)
    assert B[0].tolist() == [1, 0, 1, 1]  # -inf beats NaN; an all-NaN token keeps the lowest page; +0 beats -0
    assert np.isnan(M[0, 1]) and M[0, 0] == -inf and not np.signbit(M[0, 2]) and M[0, 3] == inf
    docs, S, ev = doc_maxsim_np(m, [0, 0, 0], 1, k=1, per_doc=3)
    assert np.isnan(S[0])
    # a NaN score ranks above every number, as in b200ms_topk
    docs, S, _ = doc_maxsim_np(np.array([[1e30], [nan]]), [0, 1], 2, k=2, per_doc=1)
    assert docs.tolist() == [1, 0]


def test_integer_sums_saturate_like_page_scores():
    m = np.full((2, 1100), 2**21, np.int64)
    docs, S, ev = doc_maxsim_np(m, [0, 1], 2, k=2, per_doc=1)
    assert S.tolist() == [I32_BOUND, I32_BOUND] and docs.tolist() == [0, 1]
    assert ev[0][1].tolist() == [1100 * 2**21]  # a share is the exact sum; the device reports it saturated


def test_documents_without_a_counted_page_are_not_returned():
    m = np.ones((4, 3))
    docs, _, _ = doc_maxsim_np(m, [0, 1, -1, 7], 3, k=5, per_doc=1, counted=[True, False, True, True])
    assert docs.tolist() == [0]
    docs, _, _ = doc_maxsim_np(np.ones((2, 0)), [0, 1], 2, k=2, per_doc=1)
    assert docs.tolist() == []  # a query without tokens finds nothing
