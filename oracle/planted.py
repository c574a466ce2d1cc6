"""oracle/planted.py -- TEST INFRASTRUCTURE ONLY: ragged corpora in which every row that matters is observable.

With random unit vectors a page's score depends on ~one row per query token out of ~1000, so a scorer that drops a row or
hands a page-boundary row to the neighbouring page is wrong only when that row happens to be some token's argmax.  Here
every page carries, for each of the D query directions, one DESIGNATED row that holds that direction's maximum by a margin
of at least 0.25 on the reference scale, for the corpus dtype the corpus is built for:

  float dtypes (bf16 / fp8 / int8): the directions are D orthonormal vectors u_d; background rows are random unit vectors in
      their orthogonal complement (dot 0 up to quantisation noise); the designated row of direction d is
      a * u_d + sqrt(1 - a^2) * (noise in the complement).
  binary: the directions are random sign patterns b_d; the designated row of d is b_d with 0 (strong) or 4 (weak) bits
      flipped; background rows are random bits, re-drawn until the margin holds.

Strengths alternate: direction d of page p is strong when (p + d) is even, weak otherwise, so the same direction is strong on
one neighbour and weak on the other -- a row given to the wrong neighbour changes a score by at least 0.35 (float) or
4/128 (binary).  Every page's strengths also carry a small per-page offset so that no two pages tie.

Designated rows sweep the positions where a scorer's bookkeeping changes: the first and last row of a page, chunk columns
0 / 31, tile columns 0 / 127 (tiles counted from the first row of the corpus), rows of a partial last chunk.  Page lengths
sweep partial chunks, 4k+1-chunk pages, pages that start in columns 0 / 32 / 64 / 96 of a 128-row tile, pages that
straddle tiles and pages longer than a 64- or 400-row work unit; empty pages sit between them.
"""
from __future__ import annotations

from dataclasses import dataclass, field
from typing import Dict, List, Sequence, Tuple

import numpy as np

from .scoring import reference_values

D = 8  # query directions: every non-empty page holds at least D rows
MARGIN = 0.25
FLOAT_STRONG, FLOAT_WEAK = 0.85, 0.50
BIN_STRONG_FLIPS, BIN_WEAK_FLIPS = 0, 4

# page lengths (>= D or 0) whose padded starts / chunk counts hit the cases listed above
BASE_LENS = [8, 9, 31, 32, 33, 0, 63, 64, 65, 95, 96, 97, 127, 128, 129, 0, 160, 161, 191, 192, 193, 255, 256, 257,
             288, 289, 400, 401, 0, 513, 700, 1030, 12, 0, 40]


@dataclass
class PlantedCorpus:
    dtype: str                       # "bf16" | "fp8" | "int8" | "binary"
    pages: List[np.ndarray]          # float32 [len, 128] each
    directions: np.ndarray           # float32 [D, 128]: u_d (float) or +-1 patterns (binary)
    designated: Dict[int, List[Tuple[int, int]]] = field(default_factory=dict)  # page -> [(row, direction)]

    @property
    def lens(self) -> List[int]:
        return [len(p) for p in self.pages]


def _page_lens(rng: np.random.Generator, n_random: int) -> List[int]:
    lens: List[int] = []
    off = 0  # padded rows so far
    for i, n in enumerate(BASE_LENS + [int(x) for x in rng.integers(D, 300, size=n_random)]):
        target = 32 * (i % 4)  # start the next page in tile column 0 / 32 / 64 / 96
        gap = (target - off) % 128
        if gap:  # a spacer page of `gap` padded rows
            spacer = gap - int(rng.integers(0, 24))
            lens.append(max(spacer, D))
            off += (lens[-1] + 31) // 32 * 32
        lens.append(n)
        off += (n + 31) // 32 * 32
    return lens


def _positions(rng: np.random.Generator, n: int, start: int) -> List[int]:
    """D distinct rows of a page of n >= D rows starting at padded corpus row `start`, boundary classes first."""
    want = [0, n - 1, 31, 32, (-start) % 128, (127 - start) % 128, (n - 1) // 32 * 32, 63, 64, 1, n - 2]
    pos: List[int] = []
    for r in want:
        if 0 <= r < n and r not in pos and len(pos) < D:
            pos.append(r)
    rest = [r for r in rng.permutation(n).tolist() if r not in pos]
    return pos + rest[: D - len(pos)]


def _strength(p: int, d: int, n_pages: int) -> float:
    base = FLOAT_STRONG if (p + d) % 2 == 0 else FLOAT_WEAK
    return base + 0.08 * p / max(n_pages, 1)  # distinct per page: no two pages tie


def planted_corpus(dtype: str, seed: int = 0, n_random: int = 40, strength_scale: float = 1.0) -> PlantedCorpus:
    """A planted corpus for `dtype`.  strength_scale < 1 weakens the plants (1.0: the documented margins; 0.0: pure
    background, the designated rows are then ordinary rows -- the control case of the sensitivity test)."""
    rng = np.random.default_rng(seed)
    lens = _page_lens(rng, n_random)
    n_pages = len(lens)
    binary = dtype == "binary"
    if binary:
        dirs = np.where(rng.random((D, 128)) < 0.5, -1.0, 1.0).astype(np.float32)
        basis_c = None
    else:
        u, _ = np.linalg.qr(rng.standard_normal((128, 128)))
        dirs = u[:, :D].T.astype(np.float32)
        basis_c = u[:, D:]

    def background(n):
        if binary:
            return np.where(rng.random((n, 128)) < 0.5, -1.0, 1.0) * rng.uniform(0.25, 1.0, size=(n, 128))
        g = rng.standard_normal((n, 128 - D)) @ basis_c.T
        return g / np.linalg.norm(g, axis=1, keepdims=True)

    pages, designated = [], {}
    start = 0
    for p, n in enumerate(lens):
        rows = background(n).astype(np.float32)
        marks = []
        if n:
            for r, d in zip(_positions(rng, n, start), rng.permutation(D).tolist()):
                if binary:
                    flips = BIN_STRONG_FLIPS if (p + d) % 2 == 0 else BIN_WEAK_FLIPS
                    row = dirs[d].copy()
                    if strength_scale < 1.0:  # control: an ordinary random row
                        row = np.where(rng.random(128) < 0.5, -1.0, 1.0)
                    elif flips:
                        row[rng.choice(128, size=flips, replace=False)] *= -1.0
                    rows[r] = row * rng.uniform(0.25, 1.0, size=128)
                else:
                    a = _strength(p, d, n_pages) * strength_scale
                    rows[r] = a * dirs[d] + np.sqrt(1.0 - a * a) * background(1)[0]
                marks.append((r, d))
            if binary and strength_scale >= 1.0:
                _redraw_binary_background(rng, rows, marks, dirs)
        designated[p] = marks
        pages.append(rows)
        start += (n + 31) // 32 * 32
    pc = PlantedCorpus(dtype, pages, dirs, designated)
    if strength_scale >= 1.0:
        check_margins(pc)
    return pc


def _redraw_binary_background(rng, rows, marks, dirs):
    marked = {r for r, _ in marks}
    for _ in range(100):
        sim = (np.sign(rows) @ np.sign(dirs).T + 128.0) / 2.0  # [n, D] 128 - hamming
        own = {d: sim[r, d] for r, d in marks}
        bad = [i for i in range(len(rows)) if i not in marked and any(sim[i, d] > own[d] - MARGIN * 128 for d in own)]
        bad += [r for r, d in marks if any(sim[r, e] > own[e] - MARGIN * 128 for e in own if e != d)]
        if not bad:
            return
        for i in set(bad) - marked:
            rows[i] = np.where(rng.random(128) < 0.5, -1.0, 1.0) * rng.uniform(0.25, 1.0, size=128)
        if set(bad) & marked:
            raise RuntimeError("two designated sign patterns are too close; use another seed")
    raise RuntimeError("could not draw a background that keeps the margin")


def direction_dots(pc: PlantedCorpus, rows: np.ndarray) -> np.ndarray:
    """[n, D] scores of rows against the D unit-scale direction tokens on the reference scale of pc.dtype."""
    if pc.dtype == "binary":
        return (np.sign(rows).astype(np.float64) @ np.sign(pc.directions).T.astype(np.float64) + 128.0) / 256.0
    return reference_values(pc.dtype, rows) @ reference_values(pc.dtype, pc.directions).T


def check_margins(pc: PlantedCorpus) -> None:
    """Every designated row is its direction's maximum on its page by >= MARGIN, on the dtype's quantised values."""
    for p, marks in pc.designated.items():
        if not marks:
            continue
        dots = direction_dots(pc, pc.pages[p])
        for r, d in marks:
            others = np.delete(dots[:, d], r)
            if others.size:
                gap = dots[r, d] - others.max()
                assert gap >= MARGIN, f"page {p} direction {d}: margin {gap:.3f} < {MARGIN}"


def planted_queries(pc: PlantedCorpus, token_counts: Sequence[int], seed: int = 1) -> List[np.ndarray]:
    """Queries whose tokens are the planted directions (scaled by c in [0.5, 1] for float dtypes, so that different
    groups of one query score differently)."""
    rng = np.random.default_rng(seed)
    out = []
    for t in token_counts:
        d = rng.integers(0, D, size=t)
        q = pc.directions[d].astype(np.float64)
        if pc.dtype != "binary":
            q = q * rng.uniform(0.5, 1.0, size=(t, 1))
        out.append(q.astype(np.float32))
    return out
