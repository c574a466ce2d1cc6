"""numpy oracle of b200ms_mmr_device, in two parts.

``page_sims`` -- sim(j -> s) of every pair of candidate slots, on the rows as the store packs them (explain_oracle.quantise):
the sum over the true rows of page j of the max over the true rows of page s of the row dot product, times score_scale,
over len_j.  Float kinds in float64 (max by fmax, as fmaxf: a NaN row counts only when every row is NaN); int8 and bits with
an exact int64 sum, then the header's fp32 steps fp32(fp32(S) * score_scale) / len_j, so the device must match them exactly.

``greedy`` -- a float32 replay of the pick rule: pick 1 by rel, every later pick by
v = fp32(fp32(lambda * rel) - fp32(fp32(1 - lambda) * red)) (numpy rounds each operation, never contracts), red the fmax of
the sims against the picks so far, in b200ms_topk's total order (-0 == +0, NaN above every number), ties to the lower slot;
lambda == 1 never reads red."""
from typing import List, Optional, Sequence

import numpy as np

from explain_oracle import quantise, similarity_np
from oracle import maxsim_oracle as orc


def quantise_rows(x: np.ndarray, kind: str) -> np.ndarray:
    """explain_oracle.quantise, with the e4m3 NaN code (0x7f / 0xff, what the packer writes for a NaN) read as NaN."""
    if kind != "fp8":
        return quantise(x, kind)
    codes = orc.quantize_e4m3_np(x, 64.0)
    nan = (codes & 0x7F) == 0x7F
    return np.where(nan, np.float32(np.nan), orc.dequantize_e4m3_np(np.where(nan, 0, codes).astype(np.uint8)))


def page_sum(dj: np.ndarray, ds: np.ndarray, kind: str):
    """S of two quantised pages: sum over the rows of dj of the max over the rows of ds (0 when either has no rows)."""
    exact = kind in ("int8", "bits")
    if len(dj) == 0 or len(ds) == 0:
        return np.int64(0) if exact else 0.0
    with np.errstate(invalid="ignore", over="ignore"):
        m = similarity_np(dj, ds, kind)
        if exact:
            return np.int64(m.max(axis=1).astype(np.int64).sum())
        return float(np.fmax.reduce(m, axis=1).sum())


def sim_value(S, len_j: int, score_scale: float, kind: str):
    """sim from S: exact kinds through the header's fp32 steps, float kinds in float64."""
    if len_j == 0:
        return np.float32(0) if kind in ("int8", "bits") else 0.0
    if kind in ("int8", "bits"):
        return np.float32(np.float32(S) * np.float32(score_scale)) / np.float32(len_j)
    return S * score_scale / len_j


def valid_slots(ids: np.ndarray, n_pages: int) -> np.ndarray:
    """Slots that name a page (0 <= id < n_pages) and are its earliest slot."""
    ids = np.asarray(ids, np.int64)
    seen, out = set(), np.zeros(len(ids), bool)
    for j, p in enumerate(ids.tolist()):
        if 0 <= p < n_pages and p not in seen:
            seen.add(p)
            out[j] = True
    return out


def page_sims(pages: Sequence[np.ndarray], ids: np.ndarray, kind: str, score_scale: float) -> np.ndarray:
    """[n_cand, n_cand] sim(slot j -> slot s) for the valid slots of one list (NaN where either slot is not valid).
    pages: the corpus's quantised pages (quantise), indexed by page id.  float64 for float kinds, float32 for exact ones."""
    ids = np.asarray(ids, np.int64)
    valid = valid_slots(ids, len(pages))
    out = np.full((len(ids), len(ids)), np.nan, dtype=np.float32 if kind in ("int8", "bits") else np.float64)
    cache = {}
    for j in np.flatnonzero(valid):
        for s in np.flatnonzero(valid):
            key = (int(ids[j]), int(ids[s]))
            if key not in cache:
                dj, ds = pages[key[0]], pages[key[1]]
                cache[key] = sim_value(page_sum(dj, ds, kind), len(dj), score_scale, kind)
            out[j, s] = cache[key]
    return out


def order_key(v: np.ndarray) -> np.ndarray:
    """b200ms_topk's total order as uint64 keys of float32 values: -0 ties +0, every NaN above +inf, NaNs tied."""
    v = np.asarray(v, np.float32) + np.float32(0)  # -0 -> +0
    u = v.view(np.uint32).astype(np.uint64)
    u = np.where(np.isnan(v), np.uint64(0x7FFFFFFF), u)
    neg = (u & np.uint64(0x80000000)) != 0
    return np.where(neg, np.uint64(0xFFFFFFFF) - u, u | np.uint64(0x80000000))


def relevance(scores: np.ndarray, q_len: int) -> np.ndarray:
    """rel = score / T_q in float32 (T_q = 0: the score)."""
    scores = np.asarray(scores, np.float32)
    return scores / np.float32(q_len) if q_len > 0 else scores.copy()


def greedy(rel: np.ndarray, sims: np.ndarray, k: int, lambda_mult: float, valid: Optional[np.ndarray] = None) -> List[int]:
    """The picked slots in pick order.  rel float32 [n]; sims [n, n] with sims[j, s] = sim(j -> s) (read as float32 only for
    the columns of picked slots); valid: the slots that may be picked (default all)."""
    rel = np.asarray(rel, np.float32)
    n = len(rel)
    live = np.ones(n, bool) if valid is None else np.asarray(valid, bool).copy()
    lam = np.float32(lambda_mult)
    one_m = np.float32(1) - lam
    red = np.full(n, np.nan, np.float32)
    picks: List[int] = []
    for i in range(k):
        if not live.any():
            break
        if i == 0 or lam == np.float32(1):
            v = rel
        else:
            with np.errstate(invalid="ignore", over="ignore"):
                v = (lam * rel) - (one_m * red)
        keys = order_key(v)
        cand = np.flatnonzero(live)
        best = cand[np.lexsort((cand, -keys[cand].astype(np.float64)))[0]]  # key DESC, slot ASC
        # lexsort on float64 of uint64 keys: keys < 2^33 are exact in float64
        picks.append(int(best))
        live[best] = False
        col = np.asarray(sims[:, best], np.float32)
        red = np.where(live, np.fmax(red, col), red)
    return picks
