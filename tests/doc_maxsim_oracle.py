"""numpy oracle of document-level MaxSim (b200ms_search_doc_maxsim_device / b200ms_rerank_doc_maxsim_batch_device).

Input: m [n_pages, T], every page's per-token maxima of ONE query (explain_oracle.maxsim_explain_np's ``best`` on the
quantised rows, so the device is compared on the same rounded inputs): float64 for bf16 / fp8, exact int64 for int8 and
bits (128 - hamming, the token constant included).  For every document D and token t:
  * M[t, D] = max over D's counted pages of m[p, t].  Floats as fmaxf: a NaN loses to any number; -0 ranks below +0.
    B[t, D] = the page holding it, the lower page on a tie (an all-NaN token: the lowest page).
  * S(D) = sum over t of M[t, D]: float64 (IEEE non-finite arithmetic), int64 saturated to +-(2^31 - 1) like the I32 sum
    rule.
  * documents ranked by S DESC (-0 == +0, NaN above every number, NaNs tied), ties to the lower ordinal; a document with
    no counted page is not ranked.
  * evidence: the distinct pages of B[:, D], each with its share (the M[t, D] it holds, added in token order), by share
    DESC in the same order, ties to the lower page.
A page counts when ``counted[p]`` (its allow bit, and it has rows) and page_doc[p] is in [0, n_docs).
"""
from typing import List, Optional, Tuple

import numpy as np

from oracle.maxsim_oracle import rank_desc_np

I32_BOUND = 2**31 - 1


def _beats(a: np.ndarray, b: np.ndarray) -> np.ndarray:
    """a strictly above b in the token-max order (fmaxf for floats; -0 < +0)."""
    if a.dtype.kind in "iu":
        return a > b
    with np.errstate(invalid="ignore"):
        zero_tie = (a == 0) & (b == 0) & ~np.signbit(a) & np.signbit(b)
        return (~np.isnan(a) & np.isnan(b)) | (a > b) | zero_tie


def doc_token_max(m: np.ndarray, page_doc, n_docs: int, counted: Optional[np.ndarray] = None
                  ) -> Tuple[np.ndarray, np.ndarray, np.ndarray]:
    """(M [n_docs, T], B int64 [n_docs, T] (-1: no counted page), found bool [n_docs])."""
    m = np.asarray(m)
    n_pages, T = m.shape
    page_doc = np.asarray(page_doc, np.int64)
    ok = (page_doc >= 0) & (page_doc < n_docs)
    if counted is not None:
        ok &= np.asarray(counted, bool)
    M = np.zeros((n_docs, T), dtype=m.dtype)
    B = np.full((n_docs, T), -1, np.int64)
    for p in np.flatnonzero(ok):  # ascending: a later page must beat the earlier one strictly
        d = int(page_doc[p])
        take = (B[d] < 0) | _beats(m[p], M[d])
        M[d] = np.where(take, m[p], M[d])
        B[d] = np.where(take, p, B[d])
    return M, B, (B >= 0).all(axis=1) & (T > 0)


def finish(s, exact: bool):
    return int(min(max(int(s), -I32_BOUND), I32_BOUND)) if exact else float(s)


def doc_scores(M: np.ndarray, found: np.ndarray) -> np.ndarray:
    """S per document (0 where not found): float64, or int64 saturated to the I32 bound."""
    exact = M.dtype.kind in "iu"
    with np.errstate(invalid="ignore", over="ignore"):
        s = M.astype(np.int64).sum(axis=1) if exact else M.sum(axis=1)
    if exact:
        s = np.clip(s, -I32_BOUND, I32_BOUND)
    return np.where(found, s, 0)


def evidence(M_d: np.ndarray, B_d: np.ndarray, per_doc: int) -> Tuple[np.ndarray, np.ndarray]:
    """(pages int64, shares) of one document, share DESC then page ASC, at most per_doc."""
    exact = M_d.dtype.kind in "iu"
    pages = np.unique(B_d)
    shares = []
    with np.errstate(invalid="ignore", over="ignore"):
        for p in pages:
            acc = np.int64(0) if exact else 0.0
            for v in M_d[B_d == p]:  # token order
                acc = acc + (np.int64(v) if exact else float(v))
            shares.append(acc)
    shares = np.array(shares, dtype=np.int64 if exact else np.float64)
    order = rank_desc_np(shares.astype(np.float64), pages)[:per_doc]
    return pages[order], shares[order]


def doc_maxsim_np(m: np.ndarray, page_doc, n_docs: int, k: int, per_doc: int, counted: Optional[np.ndarray] = None):
    """One query.  Returns (doc ids int64 [n_found <= k], scores [n_found], evidence: per document (pages, shares))."""
    M, B, found = doc_token_max(m, page_doc, n_docs, counted)
    S = doc_scores(M, found)
    docs = np.flatnonzero(found)
    order = docs[rank_desc_np(S[docs].astype(np.float64), docs)][:k]
    ev: List[Tuple[np.ndarray, np.ndarray]] = [evidence(M[d], B[d], per_doc) for d in order]
    return order.astype(np.int64), S[order], ev
