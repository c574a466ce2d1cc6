"""oracle/scoring.py -- TEST INFRASTRUCTURE ONLY.

One entry point for "what should the GPU have computed": ``oracle_scores(dtype, queries, pages)`` applies the corpus
dtype's quantisation to the float inputs exactly as the library packs them, runs the C oracle, and returns scores on the
reference scale (what ``MaxSimIndex.score_matrix`` returns).  ``TOL`` is the bar each dtype is held to:

  bf16    3e-5 relative  (same bf16-rounded inputs, fp32 accumulate: only the summation order differs)
  fp8     1e-4 relative  (dequantised e4m3 inputs; every product is exact in fp32)
  int8    exact          (integer arithmetic)
  binary  exact          (multiples of 1/128)
"""
from __future__ import annotations

from typing import Optional, Sequence

import numpy as np

from . import maxsim_oracle as orc

TOL = {"bf16": 3e-5, "fp8": 1e-4, "int8": 0.0, "binary": 0.0}
I8_SCALE = 127.0
F8_SCALE = 64.0
SCORE_QUANTUM = {"int8": 1.0 / (I8_SCALE * I8_SCALE), "binary": 1.0 / 128.0}
I32_SUM_BOUND = (1 << 31) - 1


def i32_sum(sums) -> np.ndarray:
    """The I32 sum rule of b200ms_topk: a page's exact (int64) sum of I32 group scores, clamped to +-(2^31 - 1).  This is
    what int8 and 1-bit pages are ranked by (ties at the bound break by id, or slot, like any tie)."""
    return np.clip(np.asarray(sums, np.int64), -I32_SUM_BOUND, I32_SUM_BOUND)


def i32_reported(sums, scale: float) -> np.ndarray:
    """The score reported for exact (int64) sums: float32(i32_sum(sums)) * float32(scale), rounded to float32."""
    return (i32_sum(sums).astype(np.float32) * np.float32(scale)).astype(np.float32)


def _concat(pages: Sequence[np.ndarray]) -> np.ndarray:
    live = [np.asarray(p, dtype=np.float32) for p in pages if len(p)]
    return np.concatenate(live) if live else np.zeros((0, 128), np.float32)


def reference_values(dtype: str, x: np.ndarray) -> np.ndarray:
    """The float values the scorer of `dtype` multiplies, on the reference scale (binary: +-1 per sign bit)."""
    x = np.asarray(x, dtype=np.float32)
    if dtype == "bf16":
        return orc.bf16_round_np(x).astype(np.float64)
    if dtype == "fp8":
        return orc.dequantize_e4m3_np(orc.quantize_e4m3_np(x, F8_SCALE)).astype(np.float64) / F8_SCALE
    if dtype == "int8":
        return orc.quantize_int8_np(x, I8_SCALE).astype(np.float64) / I8_SCALE
    if dtype == "binary":
        return np.where(x > 0, 1.0, -1.0)
    raise ValueError(dtype)


def oracle_scores(dtype: str, queries: Sequence[np.ndarray], pages: Sequence[np.ndarray], zero_pad_batch: int = 0) -> np.ndarray:
    """float64 [n_q, n_pages] oracle scores of the float inputs stored as `dtype`.  zero_pad_batch > 0 applies the
    zero_pad_compat clamp with batches of that many pages in list order (bf16, fp8 and int8 only)."""
    rows = _concat(pages)
    off = orc.page_offsets([len(p) for p in pages])
    zp, batch = zero_pad_batch > 0, (zero_pad_batch if zero_pad_batch > 0 else 128)
    if dtype == "binary":
        if zp:
            raise ValueError("zero_pad_compat has no 1-bit form")
        d_bits = orc.sign_pack_c(rows)
        return np.stack([orc.binary_maxsim_c(orc.sign_pack_c(q), d_bits, off)[0] for q in queries])
    if dtype == "int8":
        rq = orc.quantize_int8_np(rows, I8_SCALE)
        return np.stack([orc.int8_maxsim_c(orc.quantize_int8_np(q, I8_SCALE), rq, off, zp, batch)
                         for q in queries]).astype(np.float64) / (I8_SCALE * I8_SCALE)
    if dtype == "bf16":
        rr = orc.bf16_round_np(rows)
        return np.stack([orc.float_maxsim_c(orc.bf16_round_np(q), rr, off, zp, batch) for q in queries]).astype(np.float64)
    if dtype == "fp8":
        deq = lambda a: orc.dequantize_e4m3_np(orc.quantize_e4m3_np(a, F8_SCALE))  # noqa: E731
        rr = deq(rows)
        return np.stack([orc.float_maxsim_c(deq(q), rr, off, zp, batch) for q in queries]).astype(np.float64) / (F8_SCALE * F8_SCALE)
    raise ValueError(dtype)


def score_error(dtype: str, got: np.ndarray, want: np.ndarray) -> float:
    """Relative error (float dtypes, floor 1e-3) or the number of score quanta off (exact dtypes)."""
    got, want = np.asarray(got, np.float64), np.asarray(want, np.float64)
    if want.size == 0:
        return 0.0
    if dtype in SCORE_QUANTUM:
        q = SCORE_QUANTUM[dtype]
        return float(np.abs(np.rint(got / q) - np.rint(want / q)).max())
    return float((np.abs(got - want) / np.maximum(np.abs(want), 1e-3)).max())


def assert_scores(dtype: str, got: np.ndarray, want: np.ndarray, what: str = "") -> None:
    got, want = np.asarray(got, np.float64), np.asarray(want, np.float64)
    assert got.shape == want.shape, (what, got.shape, want.shape)
    err = score_error(dtype, got, want)
    if err > TOL[dtype]:
        if dtype in SCORE_QUANTUM:
            bad = np.argwhere(np.rint(got / SCORE_QUANTUM[dtype]) != np.rint(want / SCORE_QUANTUM[dtype]))
        else:
            bad = np.argwhere(np.abs(got - want) / np.maximum(np.abs(want), 1e-3) > TOL[dtype])
        first = tuple(int(i) for i in bad[0])
        raise AssertionError(f"{what} {dtype}: error {err:.3e} > {TOL[dtype]:.1e} at {len(bad)} entries, first {first}: "
                             f"got {got[first]!r} want {want[first]!r}")


def assert_ranking(dtype: str, got_scores: np.ndarray, got_ids: np.ndarray, got_count: int, want: np.ndarray, k: int,
                   allow: Optional[np.ndarray] = None, what: str = "") -> None:
    """One query's top-k against the oracle's (score DESC, id ASC) order of `want` [n_pages].  Exact dtypes: identical
    ids.  Float dtypes: a position may hold a different id only if the oracle scores of the two are within the tolerance
    (a near-tie that summation order may flip); the scores must match the oracle's scores of the returned ids."""
    ws, wi = orc.topk_np(want, k, allow)
    _assert_top(dtype, got_scores, got_ids, got_count, ws, wi, {}, want, what)


def slot_scores_of(want: np.ndarray, cand: np.ndarray) -> np.ndarray:
    """Oracle score of every candidate slot (0 for unused slots: -1 or an id past the corpus)."""
    cand = np.asarray(cand, dtype=np.int64)
    valid = (cand >= 0) & (cand < len(want))
    return np.where(valid, want[np.where(valid, cand, 0)], 0.0)


def assert_candidate_ranking(dtype: str, got_scores: np.ndarray, got_ids: np.ndarray, got_count: int, slot_scores: np.ndarray,
                             cand: np.ndarray, n_pages: int, k: int, what: str = "") -> None:
    """One rerank result against the oracle: the slots of `cand` that name a page (0 <= id < n_pages; -1 and ids past the
    corpus are unused slots) ordered by (oracle score of the slot DESC, slot ASC), reported as page ids."""
    cand = np.asarray(cand, dtype=np.int64)
    valid = (cand >= 0) & (cand < n_pages)
    ws, slots = orc.topk_np(np.asarray(slot_scores, np.float64), k, valid)
    by_id = {}
    for j in np.flatnonzero(valid):
        by_id.setdefault(int(cand[j]), []).append(float(slot_scores[j]))
    _assert_top(dtype, got_scores, got_ids, got_count, ws, cand[slots], by_id, None, what)


def _assert_top(dtype, got_scores, got_ids, got_count, ws, wi, by_id, want, what):
    n = len(wi)
    got_ids, got_scores = np.asarray(got_ids), np.asarray(got_scores, np.float64)
    assert int(got_count) == n, (what, int(got_count), n)
    assert np.all(got_ids[n:] == -1), what
    tol = TOL[dtype]
    if tol == 0.0:
        bad = got_ids[:n] != wi
        assert not bad.any(), (what, np.flatnonzero(bad)[:5], got_ids[:n][bad][:5], wi[bad][:5])
        assert_scores(dtype, got_scores[:n], ws, what)
        return
    for i in range(n):
        floor = max(abs(ws[i]), 1e-3)
        if got_ids[i] == wi[i]:
            assert abs(got_scores[i] - ws[i]) <= tol * floor, (what, i, int(wi[i]), got_scores[i], ws[i])
            continue
        # a near-tie that summation order may flip: the returned id's own oracle score must tie with the expected one
        own = [float(want[got_ids[i]])] if want is not None and 0 <= got_ids[i] < len(want) else by_id.get(int(got_ids[i]), [])
        assert any(abs(s - ws[i]) <= 4 * tol * floor for s in own), (what, i, int(got_ids[i]), int(wi[i]), own, ws[i])
        assert abs(got_scores[i] - ws[i]) <= 5 * tol * floor, (what, i, got_scores[i], ws[i])
