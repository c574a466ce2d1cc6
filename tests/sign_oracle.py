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
    bits: bool [padded rows, 128] in the padded page layout.  A page without rows and a query without tokens score 0.
    The products are taken in float64, which holds every one of them exactly (|q8 . row| <= 128 * 63)."""
    pm = np.where(np.asarray(bits, dtype=bool), 1.0, -1.0)
    ps = page_starts(page_lens)
    qf = [np.asarray(q8, dtype=np.float64).reshape(-1, 128) for q8 in q8s]
    out = np.zeros((len(q8s), len(page_lens)), dtype=np.int64)
    for p, n in enumerate(page_lens):
        if n <= 0:
            continue
        rows = pm[ps[p]:ps[p] + n]
        for q, q8 in enumerate(qf):
            if len(q8):
                out[q, p] = (q8 @ rows.T).max(axis=1).astype(np.int64).sum()
    return out


def topk(s: np.ndarray, k: int, allowed: Optional[np.ndarray] = None) -> List[int]:
    """Page ids of the k best by (S DESC, page id ASC) among the allowed pages (None: all)."""
    ids = np.arange(len(s)) if allowed is None else np.flatnonzero(allowed)
    order = sorted(ids.tolist(), key=lambda p: (-int(s[p]), p))
    return order[:k]


def probe_bits() -> np.ndarray:
    """bool [129, 128]: the rows of the probe corpus, one single-row page each -- page 0 has every sign negative, page
    1 + i only element i positive.  For a one-token query, S[1 + i] - S[0] = 2 q8_i (probe_q8)."""
    bits = np.zeros((129, 128), dtype=bool)
    bits[1 + np.arange(128), np.arange(128)] = True
    return bits


def probe_q8(s: np.ndarray) -> np.ndarray:
    """S [n_q, 129] of one-token queries against the probe corpus -> the q8 [n_q, 128] each query was quantised to."""
    s = np.asarray(s, dtype=np.int64).reshape(-1, 129)
    d = s[:, 1:] - s[:, :1]
    if (d % 2).any():
        raise ValueError("odd score differences: not the scores of one-token queries against the probe corpus")
    return d // 2


def tie_inputs(scale: float) -> np.ndarray:
    """float32 x with fp32(x * scale) == k + 0.5 exactly, for every k in -64 .. 63 for which such an x exists (each the one
    closest to (k + 0.5) / scale): the quantiser's rounding ties, the +-63.5 clamp boundary included."""
    s = np.float32(scale)
    out = []
    with np.errstate(over="ignore", under="ignore", invalid="ignore"):
        for k in range(-64, 64):
            t = np.float32(k + 0.5)
            x0 = np.float32(np.float64(t) / np.float64(s))
            if not np.isfinite(x0) or x0 == 0:
                continue
            cand = [x0]
            for direction in (np.float32(np.inf), np.float32(-np.inf)):
                x = x0
                for _ in range(4):
                    x = np.nextafter(x, direction, dtype=np.float32)
                    cand.append(x)
            hits = [x for x in cand if np.float32(x * s) == t]
            if hits:
                out.append(min(hits, key=lambda x: abs(np.float64(x) - np.float64(t) / np.float64(s))))
    return np.asarray(out, dtype=np.float32)


def mask_allowed(words: Optional[np.ndarray], n_pages: int) -> Optional[np.ndarray]:
    """uint32 allow words (bit p&31 of word p>>5) -> bool [n_pages]; None stays None."""
    if words is None:
        return None
    w = np.asarray(words, dtype=np.uint32).view(np.uint8)
    return np.unpackbits(w, bitorder="little")[:n_pages].astype(bool)
