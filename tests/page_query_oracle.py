"""The reference of a search whose queries are stored pages (search_pages, rerank_pages_batch, page examples), from the
packed bytes of the corpus.

    src_block(rows_u8, lens, src)            -> (query block, group offsets, query lengths): each source's true rows sliced
                                                from the packed corpus by plain indexing, the tail of its last 32-row group
                                                zero -- the block b200ms_search_pages_device should score
    page_query_reference(dtype, rows_u8, lens, src) -> float64 [n_src, n_pages]: scale_reference.reference_from_bytes of
                                                that block over every page, over the source's true length (the scale the
                                                page calls report; a source without rows scores 0)
    fuse(scores, weights)                    -> float32: an example fusion in example order, one fp32 rounding per multiply
                                                and per add, as include/b200ms.h states it

The block is built with torch slicing, never by the library's pack kernel, so a source read at a wrong offset, a tail row
left in place or a row of another page shows as a score far beyond the tolerance of oracle.scoring.
"""
from __future__ import annotations

from typing import Sequence

import numpy as np
import torch

import scale_reference as sr


def starts_of(lens: Sequence[int]) -> np.ndarray:
    """First padded row of every page (and one past the last), as the corpus lays pages out."""
    return np.concatenate([[0], np.cumsum(sr.padded_rows(lens))]).astype(np.int64)


def src_block(rows_u8: torch.Tensor, lens: Sequence[int], src: Sequence[int]):
    """Query block uint8 [32 * groups, row_bytes] on rows_u8's device, group offsets int64 [n_src + 1] and the sources' true
    lengths: source i's rows at 32 * goff[i] .. + len, zeros up to its last group's end."""
    lens = np.asarray(lens, dtype=np.int64)
    start = starts_of(lens)
    q_lens = [int(lens[p]) for p in src]
    goff = np.concatenate([[0], np.cumsum([(n + 31) // 32 for n in q_lens])]).astype(np.int64)
    block = torch.zeros((32 * int(goff[-1]), rows_u8.shape[1]), dtype=torch.uint8, device=rows_u8.device)
    for i, p in enumerate(src):
        r0 = int(start[p])
        block[32 * int(goff[i]):32 * int(goff[i]) + q_lens[i]] = rows_u8[r0:r0 + q_lens[i]]
    return block, goff, q_lens


def page_query_reference(dtype: str, rows_u8: torch.Tensor, lens: Sequence[int], src: Sequence[int],
                         budget: int = 1 << 27) -> np.ndarray:
    """float64 [n_src, n_pages]: MaxSim of every source page's packed rows against every page, on the reference scale of
    oracle.scoring (what a search reports before the division), divided by the source's true length."""
    block, goff, q_lens = src_block(rows_u8, lens, src)
    ref = sr.reference_from_bytes(dtype, rows_u8, lens, block, goff, q_lens, budget).cpu().numpy()
    n = np.asarray(q_lens, dtype=np.float64)[:, None]
    return np.where(n > 0, ref / np.maximum(n, 1.0), 0.0)


def fuse(scores: np.ndarray, weights: Sequence[float]) -> np.ndarray:
    """float32 fusion of per-example score rows scores [n_ex, n] with weights [n_ex]: acc = 0; acc = fp32(acc + fp32(w *
    s)) for every example in order."""
    s = np.asarray(scores, dtype=np.float32)
    acc = np.zeros(s.shape[1:], np.float32)
    with np.errstate(invalid="ignore", over="ignore"):
        for e, w in enumerate(weights):
            acc = (acc + (np.float32(w) * s[e]).astype(np.float32)).astype(np.float32)
    return acc
