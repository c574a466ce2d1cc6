"""numpy oracle of b200ms_explain_device: per query token, the best row of a page, the lowest row attaining it, and the whole
token x row similarity map.  It quantises with the oracle's own rules (oracle/maxsim_oracle.py), so the device is compared on
the same rounded inputs, and computes in float64 (float kinds), int64 (int8) or as 128 - hamming (bits)."""
from typing import List, Tuple

import numpy as np

from oracle import maxsim_oracle as orc

KINDS = ("bf16", "fp8", "int8", "bits")


def quantise(x: np.ndarray, kind: str, scale: float = 0.0) -> np.ndarray:
    """Rows as the store packs them, as numbers the oracle multiplies: bf16-rounded float32, e4m3 values of x * scale
    (64 by default), int8 codes of x * scale (127 by default), or the packed sign bits."""
    if kind == "bf16":
        return orc.bf16_round_np(x)
    if kind == "fp8":
        return orc.dequantize_e4m3_np(orc.quantize_e4m3_np(x, scale or 64.0))
    if kind == "int8":
        return orc.quantize_int8_np(x, scale or 127.0)
    if kind == "bits":
        return orc.sign_pack_np(x)
    raise ValueError(kind)


def similarity_np(q: np.ndarray, d: np.ndarray, kind: str) -> np.ndarray:
    """[T, P] token x row similarities of quantised operands (quantise)."""
    if kind == "bits":
        return (8 * q.shape[-1] - orc.hamming_np(q[:, None, :], d[None, :, :])).astype(np.int64)
    if kind == "int8":
        return q.astype(np.int64) @ d.astype(np.int64).T
    return q.astype(np.float64) @ d.astype(np.float64).T


def maxsim_explain_np(q: np.ndarray, rows: np.ndarray, off: np.ndarray, kind: str
                      ) -> Tuple[np.ndarray, np.ndarray, List[np.ndarray]]:
    """q [T,..] and rows [sum len,..] quantised (quantise); off = page_offsets of the pages' TRUE lengths.

    Returns (best [n_pages, T], best_row int64 [n_pages, T], maps: per page [T, len]).  best is the max over the page's rows
    and best_row the lowest row holding it; a page with no rows has best 0 and best_row -1 for every token."""
    n_pages = len(off) - 1
    T = q.shape[0]
    dt = np.float64 if kind in ("bf16", "fp8") else np.int64
    best = np.zeros((n_pages, T), dtype=dt)
    arg = np.full((n_pages, T), -1, dtype=np.int64)
    maps = []
    for p in range(n_pages):
        d = rows[off[p]:off[p + 1]]
        sim = similarity_np(q, d, kind) if d.shape[0] and T else np.zeros((T, d.shape[0]), dtype=dt)
        maps.append(sim)
        if d.shape[0] and T:
            arg[p] = sim.argmax(axis=1)  # the first (lowest) row of the max
            best[p] = sim[np.arange(T), arg[p]]
    return best, arg, maps
