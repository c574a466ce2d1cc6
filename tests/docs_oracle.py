"""numpy oracle of the grouped selection (b200ms_topk_docs / b200ms_search_docs_device / b200ms_rerank_docs_batch_device).

It walks the flat ranking of oracle/maxsim_oracle.rank_desc_np (score DESC then id ASC, -0 == +0, NaN above every number,
NaNs tied): documents come in the order of their first page in it, each with its first ``per_doc`` pages.
"""
from typing import Optional, Tuple

import numpy as np

from oracle.maxsim_oracle import rank_desc_np


def topk_docs_np(scores, page_doc, n_docs: int, k: int, per_doc: int, allow: Optional[np.ndarray] = None,
                 cand: Optional[np.ndarray] = None) -> Tuple[np.ndarray, np.ndarray, np.ndarray, int]:
    """One query.  scores: [n_items] (full scan: item p = page p; candidate mode: item j = slot j of ``cand``, page ids,
    valid in [0, len(page_doc)), where a page listed in several slots counts once, at its earliest valid slot).
    allow: bool per page (full scan).  A page is eligible when allowed and page_doc[page] is in [0, n_docs).

    Returns (pos int64 [k, per_doc]: the chosen items (-1 unused), ids int64 [k, per_doc]: their pages (-1 unused),
    page_counts int32 [k], number of documents)."""
    scores = np.asarray(scores)
    page_doc = np.asarray(page_doc, dtype=np.int64)
    n = len(scores)
    pages = np.arange(n, dtype=np.int64) if cand is None else np.asarray(cand, dtype=np.int64)
    ok = (pages >= 0) & (pages < len(page_doc))
    pg = np.where(ok, pages, 0)
    doc = np.where(ok, page_doc[pg] if len(page_doc) else -1, -1)
    ok &= (doc >= 0) & (doc < n_docs)
    if allow is not None:
        ok &= np.asarray(allow, dtype=bool)[pg]
    if cand is not None:  # later slots of a page already listed are not items of their own
        seen = set()
        for j in np.nonzero(ok)[0]:
            if pages[j] in seen:
                ok[j] = False
            seen.add(int(pages[j]))
    items = np.nonzero(ok)[0]
    flat = items[rank_desc_np(scores[items], items)]
    pos = np.full((k, per_doc), -1, dtype=np.int64)
    counts = np.zeros(k, dtype=np.int32)
    rank = {}
    for it in flat:
        d = int(doc[it])
        if d not in rank:
            if len(rank) == k:
                continue
            rank[d] = len(rank)
        r = rank[d]
        if counts[r] < per_doc:
            pos[r, counts[r]] = it
            counts[r] += 1
    ids = np.where(pos >= 0, pages[np.maximum(pos, 0)], -1)
    return pos, ids, counts, len(rank)
