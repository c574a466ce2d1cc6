"""Numpy int64 oracle of the asymmetric sign stage (include/b200ms.h, "sign candidates"): the sign rule of every corpus
dtype on the PACKED values (oracle/value_rules.py writes them), the query quantisation, the score S and the candidate order.
Test infrastructure only; the product computes all of this on the GPU."""
from __future__ import annotations

from typing import List, Optional, Sequence

import numpy as np

Q_MAX = 63


def sign_bits(dtype: str, packed: np.ndarray) -> np.ndarray:
    """Packed rows uint8 [rows, row_bytes] of corpus dtype `dtype` -> bool [rows, 128]: element > 0."""
    packed = np.ascontiguousarray(packed, dtype=np.uint8)
    if dtype == "bf16":
        v = packed.view("<u2").reshape(-1, 128).astype(np.int64)
        return (v >= 1) & (v <= 0x7F80)  # positive finite or +inf; +-0, negatives and NaN (0x7f81..0x7fff) are not
    v = packed.reshape(-1, 128).astype(np.int64)
    if dtype == "int8":
        return (v >= 1) & (v <= 0x7F)
    if dtype == "fp8":
        return (v >= 1) & (v <= 0x7E)  # e4m3: sign clear and magnitude nonzero; 0x7f is NaN
    raise ValueError(dtype)


def pack_bits(bits: np.ndarray) -> np.ndarray:
    """bool [rows, 128] -> uint8 [rows, 16], MSB first (the B1 row layout)."""
    return np.packbits(np.asarray(bits, dtype=bool).reshape(-1, 128), axis=1, bitorder="big")


def unpack_bits(rows: np.ndarray) -> np.ndarray:
    return np.unpackbits(np.asarray(rows, dtype=np.uint8).reshape(-1, 16), axis=1, bitorder="big").astype(bool)


def quantise_query(x: np.ndarray, scale: float) -> np.ndarray:
    """float32 [T, 128] -> int64 q8 = clamp(rint(fp32(x * scale)), -63, 63), ties to even, NaN -> 0, +-inf -> +-63."""
    with np.errstate(invalid="ignore", over="ignore"):
        y = np.asarray(x, dtype=np.float32).reshape(-1, 128) * np.float32(scale)
        r = np.rint(y)
    r = np.where(np.isnan(r), 0.0, np.clip(r, -Q_MAX, Q_MAX))
    return r.astype(np.int64)


def operands(q8: np.ndarray):
    """The scan's A operand and per-token constant: (2 q8, c = -sum_i q8) -- so that <2 q8, d'> + c equals the +-1 dot
    product for d' in {0, 1}."""
    q8 = np.asarray(q8, dtype=np.int64)
    return 2 * q8, -q8.sum(axis=1)


def page_starts(page_lens: Sequence[int]) -> np.ndarray:
    pad = -(-np.asarray(page_lens, dtype=np.int64) // 32) * 32
    return np.concatenate([[0], np.cumsum(pad)]).astype(np.int64)


def scores(q8s: Sequence[np.ndarray], bits: np.ndarray, page_lens: Sequence[int]) -> np.ndarray:
    """S [n_q, n_pages] int64: per query, sum over its tokens of the max over each page's TRUE rows of sum_i q8 * (+1 | -1).
    bits: bool [padded rows, 128] in the padded page layout.  A page without rows and a query without tokens score 0."""
    pm = np.where(np.asarray(bits, dtype=bool), 1, -1).astype(np.int64)
    ps = page_starts(page_lens)
    out = np.zeros((len(q8s), len(page_lens)), dtype=np.int64)
    for p, n in enumerate(page_lens):
        if n <= 0:
            continue
        rows = pm[ps[p]:ps[p] + n]
        for q, q8 in enumerate(q8s):
            if len(q8):
                out[q, p] = (np.asarray(q8, dtype=np.int64) @ rows.T).max(axis=1).sum()
    return out


def topk(s: np.ndarray, k: int, allowed: Optional[np.ndarray] = None) -> List[int]:
    """Page ids of the k best by (S DESC, page id ASC) among the allowed pages (None: all)."""
    ids = np.arange(len(s)) if allowed is None else np.flatnonzero(allowed)
    order = sorted(ids.tolist(), key=lambda p: (-int(s[p]), p))
    return order[:k]


def mask_allowed(words: Optional[np.ndarray], n_pages: int) -> Optional[np.ndarray]:
    """uint32 allow words (bit p&31 of word p>>5) -> bool [n_pages]; None stays None."""
    if words is None:
        return None
    w = np.asarray(words, dtype=np.uint32).view(np.uint8)
    return np.unpackbits(w, bitorder="little")[:n_pages].astype(bool)
