"""The work units of a filtered full scan, restated in numpy (csrc/scan_plan.cu builds them on the GPU; no GPU needed here).

    plan(masks, mask_index, page_lens, num_sms, cap) -> Plan(units, pages, rows)

masks: uint32 words, one row [ceil(n_pages/32)] or a matrix [n_masks, words]; mask_index: None (the one row filters every
query) or one row number per query, -1 = that query is unfiltered.  Units are (first chunk, end chunk) pairs in ascending
order, a chunk being 32 padded rows; pages is the ascending list of allowed pages (empty ones included: the 1-bit POPC
kernel scores those as 0), rows the padded rows of the allowed pages.

The rule: the allowed pages are the union of the masks the call's queries name (every page as soon as one query is
unfiltered), bits past n_pages ignored.  unit_rows = clamp(rows / (4 * num_sms), 128, cap), set_corpus's rule applied to
the allowed rows.  Inside every unit of the corpus' own plan (corpus_units), a filtered unit is a run of allowed pages
adjacent in memory -- pages without rows take no memory and break nothing -- cut after the page at which its rows reach
unit_rows.  So units are whole pages, never bridge a disallowed page that has rows, never cross a unit boundary of the
corpus' plan, and a mask that allows every page gives the corpus' plan back.
"""
from __future__ import annotations

from dataclasses import dataclass
from typing import List, Optional, Sequence, Tuple

import numpy as np

TILE_N = 128
CHUNK = 32


@dataclass
class Plan:
    units: List[Tuple[int, int]]
    pages: List[int]
    rows: int


def padded(page_lens: Sequence[int]) -> np.ndarray:
    lens = np.maximum(np.asarray(page_lens, dtype=np.int64), 0)
    return (lens + CHUNK - 1) // CHUNK * CHUNK


def unit_rows_for(rows: int, num_sms: int, cap: int) -> int:
    return min(max(rows // (4 * max(num_sms, 1)), TILE_N), cap)


def corpus_units(page_lens: Sequence[int], num_sms: int, cap: int) -> List[Tuple[int, int, int, int]]:
    """set_corpus's units of the whole corpus as (first chunk, end chunk, first page, end page)."""
    pad = padded(page_lens)
    ur = unit_rows_for(int(pad.sum()), num_sms, cap)
    units, acc, row, c0, p0 = [], 0, 0, 0, 0
    for p, n in enumerate(pad):
        acc += int(n)
        row += int(n)
        if acc >= ur:
            units.append((c0, row // CHUNK, p0, p + 1))
            c0, p0, acc = row // CHUNK, p + 1, 0
    if c0 != row // CHUNK:
        units.append((c0, row // CHUNK, p0, len(pad)))
    return units


def allowed_pages(masks, mask_index: Optional[Sequence[int]], n_pages: int) -> np.ndarray:
    """bool [n_pages]: the union of the mask rows the queries name."""
    m = np.ascontiguousarray(masks, dtype=np.uint32)
    if mask_index is None:
        rows = m.reshape(1, -1)
    elif any(int(i) < 0 for i in mask_index):
        return np.ones(n_pages, dtype=bool)
    else:
        rows = m.reshape(-1, (n_pages + 31) // 32)[sorted({int(i) for i in mask_index})]
    words = np.bitwise_or.reduce(rows, axis=0) if len(rows) else np.zeros((n_pages + 31) // 32, np.uint32)
    bits = (words[:, None] >> np.arange(32, dtype=np.uint32)[None, :]) & 1
    return bits.reshape(-1)[:n_pages].astype(bool)


def plan(masks, mask_index, page_lens: Sequence[int], num_sms: int, cap: int = 4096) -> Plan:
    pad = padded(page_lens)
    allow = allowed_pages(masks, mask_index, len(pad))
    rows = int(pad[allow].sum())
    ur = unit_rows_for(rows, num_sms, cap)
    start = np.concatenate([[0], np.cumsum(pad)])
    units: List[Tuple[int, int]] = []
    for _, c1, p0, p1 in corpus_units(page_lens, num_sms, cap):
        first, acc = -1, 0
        for p in range(p0, p1):
            if pad[p] == 0:
                continue
            if allow[p]:
                if first < 0:
                    first = int(start[p]) // CHUNK
                acc += int(pad[p])
                if acc >= ur:
                    units.append((first, int(start[p + 1]) // CHUNK))
                    first, acc = -1, 0
            elif first >= 0:
                units.append((first, int(start[p]) // CHUNK))
                first, acc = -1, 0
        if first >= 0:
            units.append((first, c1))
    return Plan(units, [int(p) for p in np.flatnonzero(allow)], rows)


def mask_words(allowed: np.ndarray, set_tail: bool = False) -> np.ndarray:
    """bool [n_pages] -> uint32 words; set_tail also sets the bits past n_pages in the last word."""
    allowed = np.asarray(allowed, dtype=bool)
    n = len(allowed)
    bits = np.zeros((n + 31) // 32 * 32, dtype=bool)
    bits[:n] = allowed
    if set_tail:
        bits[n:] = True
    return (bits.reshape(-1, 32).astype(np.uint32) << np.arange(32, dtype=np.uint32)).sum(axis=1).astype(np.uint32)
