"""numpy oracle of near-duplicate pages (b200ms_pair_maxsim_device, b200ms_duplicate_groups_device and the store's collapsed
search).

``pair_sims`` -- sim(a -> b) and sim(b -> a) of each pair on the quantised pages (mmr_oracle.page_sum / sim_value: float64
for the float kinds, exact int64 sums and the header's fp32 steps for int8 and bits).
``canonical_pairs`` -- (a, b) with a < b, self-pairs dropped, unique, ordered by (a, b).
``edges`` / ``union_find_labels`` -- pairs with min(sim_ab, sim_ba) >= threshold (a NaN never) and both pages allowed, and
the smallest page of each connected component (-1 for a page the mask excludes).
``collapsed_topk`` -- the best page of each group in a search's order (score DESC, page ASC), k groups at most."""
from typing import Optional, Sequence

import numpy as np

from mmr_oracle import page_sum, sim_value


def pair_sims(pages: Sequence[np.ndarray], a, b, kind: str, score_scale: float):
    """(sim_ab, sim_ba) of the pairs (a[i], b[i]) over the quantised pages; float64 for float kinds, float32 for exact."""
    dt = np.float32 if kind in ("int8", "bits") else np.float64
    sab = np.zeros(len(a), dt)
    sba = np.zeros(len(a), dt)
    for i, (x, y) in enumerate(zip(np.asarray(a).tolist(), np.asarray(b).tolist())):
        px, py = pages[x], pages[y]
        sab[i] = sim_value(page_sum(px, py, kind), len(px), score_scale, kind)
        sba[i] = sim_value(page_sum(py, px, kind), len(py), score_scale, kind)
    return sab, sba


def canonical_pairs(a, b):
    a, b = np.asarray(a, np.int64), np.asarray(b, np.int64)
    lo, hi = np.minimum(a, b), np.maximum(a, b)
    keep = lo != hi
    pairs = sorted(set(zip(lo[keep].tolist(), hi[keep].tolist())))
    return (np.array([p[0] for p in pairs], np.int64), np.array([p[1] for p in pairs], np.int64))


def edges(a, b, sab, sba, threshold: float, allowed: Optional[np.ndarray] = None):
    out = []
    for x, y, s, t in zip(np.asarray(a).tolist(), np.asarray(b).tolist(), np.asarray(sab).tolist(), np.asarray(sba).tolist()):
        if x == y or not (s >= threshold and t >= threshold):  # NaN fails
            continue
        if allowed is not None and not (allowed[x] and allowed[y]):
            continue
        out.append((x, y))
    return out


def union_find_labels(n: int, edge_list, allowed: Optional[np.ndarray] = None) -> np.ndarray:
    parent = list(range(n))

    def find(x):
        while parent[x] != x:
            parent[x] = parent[parent[x]]
            x = parent[x]
        return x

    for x, y in edge_list:
        rx, ry = find(x), find(y)
        if rx != ry:
            parent[max(rx, ry)] = min(rx, ry)
    labels = np.array([find(p) for p in range(n)], np.int64)
    # the root is the smallest member: every union points the larger root at the smaller one
    if allowed is not None:
        labels[~np.asarray(allowed, bool)] = -1
    return labels


def collapsed_topk(scores: np.ndarray, labels: np.ndarray, k: int):
    """Page ids: the best visible page (labels >= 0) of each group by (score DESC, page ASC), groups in that order."""
    order = sorted(np.flatnonzero(labels >= 0).tolist(), key=lambda p: (-float(scores[p]), p))
    seen, out = set(), []
    for p in order:
        if labels[p] in seen:
            continue
        seen.add(labels[p])
        out.append(p)
        if len(out) == k:
            break
    return out
