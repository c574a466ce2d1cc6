"""The float value rule of include/b200ms.h (hot-path section) in numpy float64, for BF16 and F8 corpora.

Inputs are PACKED values: bf16 bit patterns (uint16) or e4m3 codes (uint8), exactly what the scorer multiplies.
  * sim(q_t, d_r): every product of two packed values is exact in float64 (bf16 x bf16 needs 16 significant bits and
    exponents in [-266, 256]; e4m3 x e4m3 8 bits), and a product does not overflow or flush on its own (measured on an
    H100: 2^64 * 2^64 + (-2^64) * 2^64 in one MMA step is 0).  The products are summed with IEEE non-finite arithmetic
    (NaN if a NaN occurs or +inf meets -inf, else +-inf if one occurs); a finite sum is taken in float64 and rounded to
    fp32 once: to nearest even in fp32's normal range, past it to +-inf, and into its subnormal range (below 2^-126) toward
    zero, to a multiple of 2^-149, as the H100's tensor core does (measured on single bf16 products: 1.0078 * 2^-150 gives
    0, 1.5 * 2^-149 gives 2^-149, where round-to-nearest would give 2^-149 and 2^-148).
  * The max over a page's rows is fmaxf's: NaN only when every row is NaN.
  * A query's score is the IEEE sum of its true tokens' maxima, rounded to fp32; a page without rows scores 0.
  * zero_pad_compat: a clamped page's token max m becomes fmaxf(m, 0).
The tensor core adds in fp32 in an order of its own, so a finite result may differ from this one by rounding (TOL of
oracle/scoring.py); a single nonzero product, the probes' case, has no rounding order to differ in.
"""
from __future__ import annotations

from typing import Optional, Sequence

import numpy as np

from oracle import maxsim_oracle as orc

F8_SCALE = 64.0  # MaxSimIndex's e4m3 scale: reference-scale scores are raw / F8_SCALE^2


def bf16_values(bits) -> np.ndarray:
    """bf16 bit patterns -> float64 (every pattern: subnormals, +-0, +-inf and NaN included)."""
    b = np.asarray(bits, dtype=np.uint16).astype(np.uint32) << 16
    with np.errstate(invalid="ignore"):
        return b.view(np.float32).astype(np.float64)


def e4m3_values(codes) -> np.ndarray:
    """e4m3 codes -> float64: 0x7f and 0xff are NaN (e4m3 has no infinity), every other code its finite value."""
    c = np.asarray(codes, dtype=np.uint8)
    nan = (c & 0x7F) == 0x7F
    v = orc.dequantize_e4m3_np(np.where(nan, 0, c)).astype(np.float64)
    return np.where(nan, np.nan, v)


def packed_values(dtype: str, packed: np.ndarray) -> np.ndarray:
    """Packed rows [n, row bytes] (uint8, the corpus layout) -> float64 [n, 128]."""
    packed = np.ascontiguousarray(packed, dtype=np.uint8)
    if dtype == "bf16":
        return bf16_values(packed.reshape(-1, 128, 2).view(np.uint16)[..., 0])
    if dtype == "fp8":
        return e4m3_values(packed.reshape(-1, 128))
    raise ValueError(dtype)


def pack_values(dtype: str, x: np.ndarray) -> np.ndarray:
    """Float inputs (float32 or bfloat16 values as float32) -> the packed values b200ms_pack_pages / pack_queries store,
    as float64: bf16 round-to-nearest-even; e4m3 of x * F8_SCALE (saturating: +-inf -> +-448, NaN -> 0x7f)."""
    x = np.asarray(x, dtype=np.float32)
    if dtype == "bf16":
        return orc.bf16_round_np(x).astype(np.float64)
    if dtype == "fp8":
        return e4m3_values(orc.quantize_e4m3_np(x, F8_SCALE))
    raise ValueError(dtype)


LEAST_SUBNORMAL = 2.0 ** -149


def fp32(x) -> np.ndarray:
    """float64 -> fp32 under the value rule, as float64: round to nearest even in the normal range, +-inf past it, and
    toward zero to a multiple of 2^-149 below 2^-126 (the tensor core's subnormal results)."""
    x = np.asarray(x, dtype=np.float64)
    with np.errstate(over="ignore", invalid="ignore"):
        rn = x.astype(np.float32).astype(np.float64)
        return np.where(np.abs(x) < 2.0 ** -126, np.trunc(x / LEAST_SUBNORMAL) * LEAST_SUBNORMAL, rn)


def ieee_sum(terms: np.ndarray, axis: int = -1) -> np.ndarray:
    """Sum along `axis` with IEEE non-finite rules and one fp32 rounding of a finite result."""
    t = np.asarray(terms, dtype=np.float64)
    nan = np.isnan(t).any(axis=axis)
    pinf = (t == np.inf).any(axis=axis)
    ninf = (t == -np.inf).any(axis=axis)
    finite = fp32(np.where(np.isfinite(t), t, 0.0).sum(axis=axis))
    out = np.where(pinf, np.inf, np.where(ninf, -np.inf, finite))
    return np.where(nan | (pinf & ninf), np.nan, out)


def _similarities_elementwise(q: np.ndarray, d: np.ndarray) -> np.ndarray:
    with np.errstate(invalid="ignore", over="ignore"):
        prod = q[:, None, :] * d[None, :, :]
    return ieee_sum(prod, axis=-1)


def similarities(q: np.ndarray, d: np.ndarray) -> np.ndarray:
    """[T, 128] x [R, 128] packed values -> [T, R] sim(q_t, d_r) under the rule: the finite part is one float64 matrix
    product, the non-finite products are counted with 0/1 matrix products (the same as _similarities_elementwise, faster)."""
    q, d = np.asarray(q, np.float64), np.asarray(d, np.float64)
    qf, df = np.where(np.isfinite(q), q, 0.0), np.where(np.isfinite(d), d, 0.0)
    finite = fp32(qf @ df.T)
    f = lambda m: m.astype(np.float64)  # noqa: E731
    qn, dn = f(np.isnan(q)), f(np.isnan(d))
    qpi, qni, dpi, dni = f(q == np.inf), f(q == -np.inf), f(d == np.inf), f(d == -np.inf)
    qz, dz = f(q == 0), f(d == 0)
    qp, qm, dp, dm = f(q > 0), f(q < 0), f(d > 0), f(d < 0)
    one_q, one_d = np.ones_like(qn), np.ones_like(dn)
    nan = (qn @ one_d.T + one_q @ dn.T + qz @ (dpi + dni).T + (qpi + qni) @ dz.T) > 0
    pos = (qpi @ dp.T + qni @ dm.T + qp @ dpi.T + qm @ dni.T) > 0
    neg = (qpi @ dm.T + qni @ dp.T + qp @ dni.T + qm @ dpi.T) > 0
    out = np.where(pos, np.inf, np.where(neg, -np.inf, finite))
    return np.where(nan | (pos & neg), np.nan, out)


def fmax_rows(sims: np.ndarray) -> np.ndarray:
    """[T, R] -> [T]: fmaxf over the rows (NaN only when every row is NaN).  R must be > 0."""
    s = np.asarray(sims, np.float64)
    all_nan = np.isnan(s).all(axis=1)
    return np.where(all_nan, np.nan, np.where(np.isnan(s), -np.inf, s).max(axis=1, initial=-np.inf))


def token_maxima(q: np.ndarray, d: np.ndarray, clamp: bool = False) -> np.ndarray:
    """Per true token of q: its max over the rows of page d (clamp: fmaxf(max, 0), the zero_pad_compat rule)."""
    m = fmax_rows(similarities(q, d))
    return np.where(np.isnan(m), 0.0, np.maximum(m, 0.0)) if clamp else m


def page_score(q: np.ndarray, d: np.ndarray, clamp: bool = False) -> float:
    """A query's score on one page: the IEEE sum of its tokens' maxima rounded to fp32; a page without rows scores 0."""
    if len(d) == 0 or len(q) == 0:
        return 0.0
    return float(ieee_sum(token_maxima(q, d, clamp)))


def scores(queries: Sequence[np.ndarray], pages: Sequence[np.ndarray], clamp: Optional[Sequence[bool]] = None) -> np.ndarray:
    """[n_q, n_pages] page_score of every pair, in packed units (divide by F8_SCALE^2 for an fp8 corpus's reference scale).
    clamp[p]: the zero_pad_compat clamp applies to page p."""
    lens = [len(q) for q in queries]
    qcat = np.concatenate([np.asarray(q, np.float64) for q in queries]) if queries else np.zeros((0, 128))
    seg = np.cumsum([0] + lens)
    out = np.zeros((len(queries), len(pages)))
    for p, d in enumerate(pages):
        if len(d) == 0:
            continue
        m = fmax_rows(similarities(qcat, d))
        if clamp is not None and clamp[p]:
            m = np.where(np.isnan(m), 0.0, np.maximum(m, 0.0))
        for i in range(len(queries)):
            out[i, p] = ieee_sum(m[seg[i]:seg[i + 1]]) if lens[i] else 0.0
    return out


def zero_pad_clamped(lens: Sequence[int], batch: int) -> np.ndarray:
    """zero_pad_compat: which pages (in list order, batches of `batch`) are shorter than the longest page of their batch."""
    lens = np.asarray(lens, dtype=np.int64)
    out = np.zeros(len(lens), dtype=bool)
    for b in range(0, len(lens), batch):
        seg = lens[b:b + batch]
        out[b:b + batch] = seg < seg.max()
    return out
