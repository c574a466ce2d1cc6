"""The window walk of b200ms_compact_rows, restated in numpy (csrc/compact.cu runs it on the GPU; no GPU needed here).

    compact_in_place(buf, row_bytes, run_start, run_rows, ...) -> list of windows (first row, rows, "direct" | "bounce")

Runs of rows, ascending and disjoint, move down inside `buf` until they are contiguous from row 0.  src(d), the source row of
destination row d, ascends with d and src(d) >= d.  The destination is walked in ascending windows, each a launch of its own
that ends before the next begins:

  * rows already in place (leading runs that start at their destination) are skipped;
  * at the window's first row d0 the displacement is disp = src(d0) - d0, and every source of [d0, d0 + n) lies at or past
    d0 + disp.  disp >= min_direct_rows: a DIRECT window of n = min(disp, max_direct_rows) rows, gathered straight into
    place -- its sources lie at or past its end, so the order in which the launch's threads run does not matter;
  * else a BOUNCE window of at most window_rows rows: gathered into a bounce buffer, then copied out.

The model keeps a flag per row of `buf`, set when a launch writes the row, and asserts that no launch reads a flagged row:
a direct window flags its destination BEFORE its reads are checked (its threads run in any order), a bounce window after.
The library's constants are 64 MiB windows, direct from a quarter of that, at most 1 GiB per direct window; the tests pass
small ones so that every case crosses many windows.
"""
from __future__ import annotations

from typing import List, Sequence, Tuple

import numpy as np

WINDOW_BYTES = 64 << 20
MIN_DIRECT_BYTES = WINDOW_BYTES // 4
MAX_DIRECT_BYTES = WINDOW_BYTES * 16


def library_windows(row_bytes: int) -> Tuple[int, int, int]:
    """(window_rows, min_direct_rows, max_direct_rows) the library uses for rows of `row_bytes`."""
    return WINDOW_BYTES // row_bytes, -(-MIN_DIRECT_BYTES // row_bytes), MAX_DIRECT_BYTES // row_bytes


def check_runs(run_start: Sequence[int], run_rows: Sequence[int]) -> None:
    end = 0
    for i, (s, n) in enumerate(zip(run_start, run_rows)):
        if n < 0 or s < end:
            raise ValueError(f"run {i} is negative, overlaps the run before it or is out of order")
        end = s + n


def out_of_place(buf: np.ndarray, row_bytes: int, run_start: Sequence[int], run_rows: Sequence[int]) -> np.ndarray:
    """The runs copied into a second buffer: what the in-place walk must leave in the first rows of `buf`."""
    rows = buf.reshape(-1, row_bytes)
    parts = [rows[s:s + n] for s, n in zip(run_start, run_rows)]
    return np.concatenate(parts) if parts else rows[:0].copy()


def compact_in_place(buf: np.ndarray, row_bytes: int, run_start: Sequence[int], run_rows: Sequence[int], window_rows: int,
                     min_direct_rows: int, max_direct_rows: int) -> List[Tuple[int, int, str]]:
    check_runs(run_start, run_rows)
    rows = buf.reshape(-1, row_bytes)  # a view: the walk writes into buf
    start = np.asarray(run_start, dtype=np.int64)
    pre = np.concatenate([[0], np.cumsum(np.asarray(run_rows, dtype=np.int64))]).astype(np.int64)
    n_runs, total = len(start), int(pre[-1])
    written = np.zeros(rows.shape[0], dtype=bool)
    windows: List[Tuple[int, int, str]] = []
    r = 0
    while r < n_runs and start[r] == pre[r]:
        r += 1
    if r == n_runs:
        return windows
    d = int(pre[r])
    while d < total:
        r_lo = int(np.searchsorted(pre, d, side="right")) - 1  # the last run with pre <= d: never an empty one
        disp = int(start[r_lo] + (d - pre[r_lo]) - d)
        direct = disp >= min_direct_rows
        n = min(min(disp, max_direct_rows) if direct else window_rows, total - d)
        dst = np.arange(d, d + n, dtype=np.int64)
        run = np.searchsorted(pre, dst, side="right") - 1
        src = start[run] + (dst - pre[run])
        if direct:
            written[dst] = True
            assert not written[src].any(), f"direct window at row {d} reads rows a launch has overwritten"
            rows[dst] = rows[src]
        else:
            assert not written[src].any(), f"bounce window at row {d} reads rows a launch has overwritten"
            bounce = rows[src].copy()
            rows[dst] = bounce
            written[dst] = True
        windows.append((d, n, "direct" if direct else "bounce"))
        d += n
    return windows
