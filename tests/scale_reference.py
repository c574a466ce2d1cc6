"""Planted corpora of any size built on the GPU, and the float64 MaxSim reference of what the scan should return on them.

    build(dtype, n_pages, seed)                              -> MaxSimIndex with the corpus packed by the library itself
    reference_scores(idx, q_packed, group_offsets, q_lens)  -> float64 [n_q, n_pages] on the score_matrix scale
    sign_rows_of(dtype, rows_u8) / sign_reference(...)     -> the sign stage's sign rows and its exact integer S

Corpus (generate_chunks): page lengths are mostly 1000 .. 1100 rows, with pages of 1 .. 1025 rows hitting the chunk and tile
edges (31 / 32 / 33, 127 / 128 / 129) every 61st page and runs of four empty pages, so the corpora reach a few GB at a few
ten thousand pages.  As in oracle/planted.py every page carries, for each of D query directions, one designated row that holds
that direction's maximum by at least planted.MARGIN (a page of n < D rows carries n of them).  Designated rows sweep the first
and last row of the page, chunk columns 0 / 31 and tile columns 0 / 127 (tiles counted from the first row of the corpus), so a
row handed to the wrong page, dropped or read at a wrong offset moves a score far beyond the tolerance.  Float dtypes: the
directions u_d are orthonormal, background rows are unit rows with dot BACKGROUND_DOT to every direction (the rest in the
directions' orthogonal complement), designated rows are a * u_d + sqrt(1-a^2) * background; binary: the directions are sign patterns at least 44 bits apart, designated rows carry 0 or 4 flipped bits and
background rows are redrawn until the margin holds.

Reference: it decodes the packed bytes the scan itself reads (idx.packed_rows() and the packed query block of score_groups),
true rows only -- bf16 exactly, int8 as integers, e4m3 through a 256-entry table, 1-bit as +-1 with 128 - ham = (dot + 128) / 2
-- then multiplies per chunk of pages, takes each page's maximum per token and sums a query's tokens.  Pages without rows
score 0.  int8, fp8 and 1-bit results are exact: float64 holds every product and every sum exactly.  bf16 is within rounding
of exact.  The 1-bit products are taken in float16 on the GPU: every operand is +-1 and every partial sum an integer of
magnitude <= 128, which float16 holds exactly, so the result does not depend on the accumulation order or width.  The same
code runs on CPU tensors (tests/test_scale_reference_cpu.py ties it to oracle.scoring.oracle_scores).
"""
from __future__ import annotations

from typing import Iterator, List, Optional, Sequence, Tuple

import numpy as np
import torch

from oracle import planted
from oracle.scoring import F8_SCALE, I8_SCALE

D = planted.D
ROW_BYTES = {"bf16": 256, "int8": 128, "fp8": 128, "binary": 16}
EDGE_LENS = [1, 2, 7, 8, 31, 32, 33, 63, 64, 65, 127, 128, 129, 1023, 1024, 1025]
CHUNK_PAGES = 2048  # pages generated and packed per add_pages call
# float background rows: this dot product with every direction, so that a token no designated row of a page answers still
# scores well above the float32 rounding of its 128 products (a score near 0 would leave the relative tolerance nothing)
BACKGROUND_DOT = 0.05
BIN_MIN_DIR_DISTANCE = 44  # bits between two direction patterns: a weak designated row (4 flips) stays 36+ bits off the others


# ------------------------------------------------------------------------------------------------ corpus
def page_lens(n_pages: int, seed: int) -> np.ndarray:
    """int64 [n_pages]: mostly 1000 .. 1100 rows; every 61st page an edge length; runs of four empty pages every 997 pages."""
    rng = np.random.default_rng(seed)
    lens = rng.integers(1000, 1101, size=n_pages).astype(np.int64)
    i = np.arange(n_pages)
    edge = i % 61 == 30
    lens[edge] = np.asarray(EDGE_LENS)[(i[edge] // 61) % len(EDGE_LENS)]
    lens[(i % 997) >= 993] = 0
    return lens


def padded_rows(lens) -> np.ndarray:
    return (np.asarray(lens, dtype=np.int64) + 31) // 32 * 32


def designated_positions(lens: np.ndarray, starts: np.ndarray) -> np.ndarray:
    """int64 [n_pages, D]: the designated rows of every page (-1 past min(len, D)), boundary classes first: first and last
    row, chunk columns 31 / 0 (rows 31, 32), tile columns 0 / 127, the first row of the last chunk, then rows 1, 2, ..."""
    n = np.asarray(lens, dtype=np.int64)[:, None]
    s = np.asarray(starts, dtype=np.int64)[:, None]
    cand = np.concatenate([np.zeros_like(n), n - 1, np.full_like(n, 31), np.full_like(n, 32), (-s) % 128, (127 - s) % 128,
                           (n - 1) // 32 * 32, np.broadcast_to(np.arange(1, D + 1), (len(n), D))], axis=1)
    ok = (cand >= 0) & (cand < n)
    for j in range(1, cand.shape[1]):  # keep the first occurrence of each row
        ok[:, j] &= ~((cand[:, :j] == cand[:, j:j + 1]) & ok[:, :j]).any(axis=1)
    order = np.argsort(~ok, axis=1, kind="stable")[:, :D]
    pos = np.take_along_axis(cand, order, axis=1)
    return np.where(np.take_along_axis(ok, order, axis=1), pos, -1)


def directions(dtype: str, seed: int) -> Tuple[np.ndarray, Optional[np.ndarray]]:
    """(float32 [D, 128] query directions, float64 [128, 128 - D] basis of their complement or None for binary)."""
    rng = np.random.default_rng(seed)
    if dtype == "binary":
        while True:
            dirs = np.where(rng.random((D, 128)) < 0.5, -1.0, 1.0)
            dist = (128.0 - dirs @ dirs.T) / 2.0
            if dist[~np.eye(D, dtype=bool)].min() >= BIN_MIN_DIR_DISTANCE:
                return dirs.astype(np.float32), None
    u, _ = np.linalg.qr(rng.standard_normal((128, 128)))
    return u[:, :D].T.astype(np.float32), u[:, D:]


def _strength(pages: torch.Tensor, d: torch.Tensor, n_pages: int) -> torch.Tensor:
    base = torch.where((pages[:, None] + d) % 2 == 0, planted.FLOAT_STRONG, planted.FLOAT_WEAK)
    return base + 0.08 * pages[:, None].double() / max(n_pages, 1)  # distinct per page


def generate_chunks(dtype: str, n_pages: int, seed: int, device) -> Iterator[Tuple[int, np.ndarray, torch.Tensor, np.ndarray, np.ndarray]]:
    """Yields (first page, lens [n], rows float32 [sum lens, 128] on `device`, designated rows [n, D] (-1 unused), their
    directions [n, D]) for consecutive chunks of CHUNK_PAGES pages."""
    device = torch.device(device)
    lens = page_lens(n_pages, seed)
    starts = np.concatenate([[0], np.cumsum(padded_rows(lens))])[:-1]
    pos_all = designated_positions(lens, starts)
    dirs_np, basis = directions(dtype, seed + 1)
    dirs = torch.from_numpy(dirs_np).to(device)
    basis_t = None if basis is None else torch.from_numpy(basis.T.astype(np.float32)).to(device)  # [128 - D, 128]
    g = torch.Generator(device=device).manual_seed(seed + 2)
    rng = np.random.default_rng(seed + 3)
    for p0 in range(0, n_pages, CHUNK_PAGES):
        p1 = min(p0 + CHUNK_PAGES, n_pages)
        ln = lens[p0:p1]
        total = int(ln.sum())
        pos = pos_all[p0:p1]
        dir_of = np.argsort(rng.random((p1 - p0, D)), axis=1)  # a permutation of the directions per page
        first = np.concatenate([[0], np.cumsum(ln)])[:-1]
        used = pos >= 0
        flat_rows = torch.from_numpy((first[:, None] + pos)[used]).to(device)
        flat_dirs = torch.from_numpy(dir_of[used]).to(device)
        flat_pages = torch.from_numpy(np.broadcast_to(np.arange(p0, p1)[:, None], pos.shape)[used].copy()).to(device)
        if dtype == "binary":
            rows = _binary_rows(total, flat_rows, flat_dirs, flat_pages, dirs, torch.from_numpy(ln).to(device), p0, g)
        else:
            rows = torch.randn((total, 128 - D), generator=g, device=device) @ basis_t
            rows = torch.nn.functional.normalize(rows, dim=1) * (1.0 - D * BACKGROUND_DOT ** 2) ** 0.5
            rows += BACKGROUND_DOT * dirs.sum(dim=0)  # unit rows, BACKGROUND_DOT along every direction
            a = _strength(flat_pages, flat_dirs[:, None], n_pages)[:, 0].float()
            rows[flat_rows] = a[:, None] * dirs[flat_dirs] + torch.sqrt(1.0 - a * a)[:, None] * rows[flat_rows]
        yield p0, ln, rows, pos, dir_of


def _binary_rows(total, flat_rows, flat_dirs, flat_pages, dirs, lens_t, p0, g):
    """Random +-1 rows with magnitudes in [0.25, 1]; designated rows are their direction with 0 (strong) or 4 (weak) bits
    flipped; background rows within MARGIN * 128 bits of a designated row's similarity to its direction are redrawn."""
    device = dirs.device

    def draw(n):
        sign = torch.where(torch.rand((n, 128), generator=g, device=device) < 0.5, -1.0, 1.0)
        return sign * (0.25 + 0.75 * torch.rand((n, 128), generator=g, device=device))

    rows = draw(total)
    weak = ((flat_pages + flat_dirs) % 2 == 1)
    plant = dirs[flat_dirs].clone()
    flips = torch.argsort(torch.rand((len(flat_dirs), 128), generator=g, device=device), dim=1)[:, :planted.BIN_WEAK_FLIPS]
    sign = torch.ones_like(plant)
    sign.scatter_(1, flips, -1.0)
    plant = torch.where(weak[:, None], plant * sign, plant)
    rows[flat_rows] = plant * (0.25 + 0.75 * torch.rand(plant.shape, generator=g, device=device))
    page_of_row = torch.repeat_interleave(torch.arange(len(lens_t), device=device), lens_t)
    designated = torch.zeros(total, dtype=torch.bool, device=device)
    designated[flat_rows] = True
    # threshold[page, d]: the designated row's similarity minus the margin (+inf where the page has no row for d)
    sims = (torch.sign(rows[flat_rows]) * dirs[flat_dirs]).sum(dim=1)
    thr = torch.full((len(lens_t), D), float("inf"), device=device)
    thr[flat_pages - p0, flat_dirs] = (sims + 128.0) / 2.0 - planted.MARGIN * 128.0
    for _ in range(100):
        sim = (torch.sign(rows) @ dirs.T + 128.0) / 2.0  # [total, D] = 128 - hamming
        bad = ((sim > thr[page_of_row]).any(dim=1) & ~designated).nonzero()[:, 0]
        if len(bad) == 0:
            return rows
        rows[bad] = draw(len(bad))
    raise RuntimeError("could not draw a binary background that keeps the margin")


def build(dtype: str, n_pages: int, seed: int, device: int = 0, **index_kw):
    """MaxSimIndex of the planted corpus: one exact allocation (reserve_rows), then add_pages of device tensors chunk by
    chunk, so the pack kernel writes the layout (pad rows repeat the page's last true row)."""
    from morphik_core_b200.index import MaxSimIndex

    idx = MaxSimIndex(device=device, dtype=dtype, **index_kw)
    idx.reserve_rows(int(padded_rows(page_lens(n_pages, seed)).sum()))
    for _, ln, rows, _, _ in generate_chunks(dtype, n_pages, seed, idx.device):
        off = np.concatenate([[0], np.cumsum(ln)])
        idx.add_pages([rows[off[i]:off[i + 1]] for i in range(len(ln))])
        del rows
    idx._attach()
    return idx


def queries(dtype: str, seed: int, token_counts: Sequence[int], q_seed: int = 1) -> List[np.ndarray]:
    """Queries whose tokens are the corpus' planted directions (float dtypes: scaled by c in [0.5, 1])."""
    pc = planted.PlantedCorpus(dtype, [], directions(dtype, seed + 1)[0])
    return planted.planted_queries(pc, token_counts, seed=q_seed)


# ------------------------------------------------------------------------------------------------ reference
def e4m3_table() -> torch.Tensor:
    """float64 [256]: the value of every e4m3 code (0x7f / 0xff: NaN)."""
    code = torch.arange(256, dtype=torch.int64)
    e, m = (code >> 3) & 0xF, (code & 7).double()
    mag = torch.where(e == 0, m / 8.0 * 2.0 ** -6, (1.0 + m / 8.0) * torch.pow(2.0, (e - 7).double()))
    mag = torch.where((code & 0x7F) == 0x7F, torch.full_like(mag, float("nan")), mag)
    return torch.where(code >= 128, -mag, mag)


_SHIFTS = torch.arange(7, -1, -1, dtype=torch.uint8)


def unpack_bits(raw: torch.Tensor) -> torch.Tensor:
    """uint8 [n, 16] MSB-first sign bits -> uint8 [n, 128] of 0 / 1."""
    return ((raw[:, :, None] >> _SHIFTS.to(raw.device)) & 1).reshape(raw.shape[0], 128)


def decode(dtype: str, raw: torch.Tensor, out_dtype=torch.float64) -> torch.Tensor:
    """Packed rows uint8 [n, row_bytes] -> [n, 128] values the scan multiplies (int8 codes, e4m3 values, +-1 for bits)."""
    if dtype == "bf16":
        return raw.view(torch.bfloat16).to(out_dtype)
    if dtype == "int8":
        return raw.view(torch.int8).to(out_dtype)
    if dtype == "fp8":
        return e4m3_table().to(raw.device)[raw.long()].to(out_dtype)
    if dtype == "binary":
        return (unpack_bits(raw).to(out_dtype) * 2 - 1)
    raise ValueError(dtype)


def _score_divisor(dtype: str) -> float:
    """Raw sums / this = scores on the reference scale (as oracle.scoring divides)."""
    return {"bf16": 1.0, "int8": I8_SCALE * I8_SCALE, "fp8": F8_SCALE * F8_SCALE, "binary": 128.0}[dtype]


def reference_from_bytes(dtype: str, rows_u8: torch.Tensor, lens: Sequence[int], q_u8: torch.Tensor, group_offsets,
                         q_lens: Sequence[int], budget: int = 1 << 27) -> torch.Tensor:
    """float64 [n_q, n_pages] MaxSim of the packed query block q_u8 [>= 32 * groups, row_bytes] (query q's token j at row
    32 * group_offsets[q] + j) against the packed corpus rows_u8 [rows_padded, row_bytes] of pages of `lens` true rows
    (each padded to whole 32-row chunks), on the score_matrix scale.  `budget` caps the token x row products per step."""
    goff = np.asarray(group_offsets, dtype=np.int64)
    tok = np.concatenate([32 * goff[q] + np.arange(int(t)) for q, t in enumerate(q_lens)] + [np.zeros(0, np.int64)])
    binary = dtype == "binary"
    cdt = torch.float16 if binary and rows_u8.device.type == "cuda" else torch.float64
    q = decode(dtype, q_u8[torch.from_numpy(tok).to(q_u8.device)].to(rows_u8.device), cdt)  # [T, 128]
    out = _page_maxsim(q, lambda r0, r1: decode(dtype, rows_u8[r0:r1], cdt), lens, q_lens, rows_u8.device, budget,
                       (lambda m: (m + 128.0) / 2.0) if binary else None)  # 1-bit: 128 - hamming
    return out / _score_divisor(dtype)


def _page_maxsim(q: torch.Tensor, rows_of, lens: Sequence[int], q_lens: Sequence[int], device, budget: int,
                 chunk_map=None) -> torch.Tensor:
    """float64 [n_q, n_pages]: per query (q_lens consecutive tokens of q [T, 128]), the sum over its tokens of the max over
    each page's true rows of q . row, with rows_of(r0, r1) the padded rows [r0, r1) as q's dtype.  chunk_map: applied to the
    per-chunk maxima (float64).  Pages without rows and queries without tokens score 0."""
    lens_np = np.asarray(lens, dtype=np.int64)
    n_pages, n_q = len(lens_np), len(q_lens)
    tok_query = torch.from_numpy(np.repeat(np.arange(n_q), np.asarray(q_lens, dtype=np.int64))).to(device)
    T = q.shape[0]
    out = torch.zeros((n_q, n_pages), dtype=torch.float64, device=device)
    if T == 0 or n_pages == 0:
        return out
    pad = padded_rows(lens_np)
    start = np.concatenate([[0], np.cumsum(pad)])
    rows_per_step = min(max(budget // T, 1100), 1 << 20)
    p0 = 0
    while p0 < n_pages:
        p1 = int(np.searchsorted(start, start[p0] + rows_per_step, side="right")) - 1
        p1 = min(max(p1, p0 + 1), n_pages)
        r0, r1 = int(start[p0]), int(start[p1])
        if r1 > r0:
            x = rows_of(r0, r1)  # the chunk's padded rows; the pad rows are masked below
            sim = q @ x.T  # [T, R]
            col = np.arange(r1 - r0) + r0
            page_of_row = np.repeat(np.arange(p0, p1), pad[p0:p1])
            is_pad = torch.from_numpy(col - start[page_of_row] >= lens_np[page_of_row]).to(device)
            sim.masked_fill_(is_pad[None, :], float("-inf"))
            chunk_max = sim.view(T, -1, 32).amax(dim=2).double()  # per 32-row chunk: every page owns whole chunks
            if chunk_map is not None:
                chunk_max = chunk_map(chunk_max)
            chunk_page = torch.from_numpy(page_of_row[::32] - p0).to(device)
            best = torch.zeros((T, p1 - p0), dtype=torch.float64, device=device)
            best.scatter_reduce_(1, chunk_page[None, :].expand(T, -1), chunk_max, "amax", include_self=False)
            out[:, p0:p1].index_add_(0, tok_query, best)
            del sim, chunk_max, best, x
        p0 = p1
    return out


# ------------------------------------------------------------------------------------------------ sign stage
_BIT_WEIGHTS = torch.tensor([128, 64, 32, 16, 8, 4, 2, 1], dtype=torch.int32)


def sign_rows_of(dtype: str, rows_u8: torch.Tensor, step: int = 1 << 20) -> torch.Tensor:
    """uint8 [n, 16]: the sign rows of packed rows uint8 [n, row_bytes] by the header's rule on the packed values (bf16
    0x0001 .. 0x7f80, int8 1 .. 127, e4m3 0x01 .. 0x7e), MSB first, with torch integer ops, `step` rows at a time."""
    out = torch.empty((rows_u8.shape[0], 16), dtype=torch.uint8, device=rows_u8.device)
    w = _BIT_WEIGHTS.to(rows_u8.device)
    for r0 in range(0, rows_u8.shape[0], step):
        raw = rows_u8[r0:r0 + step]
        if dtype == "bf16":
            v = raw.view(torch.int16).to(torch.int32) & 0xFFFF
            bits = (v >= 1) & (v <= 0x7F80)
        else:
            v = raw.to(torch.int32)
            bits = (v >= 1) & (v <= {"int8": 0x7F, "fp8": 0x7E}[dtype])
        out[r0:r0 + step] = (bits.view(-1, 16, 8).to(torch.int32) * w).sum(dim=2).to(torch.uint8)
    return out


def sign_reference(sign_rows: torch.Tensor, lens: Sequence[int], q8s: Sequence[np.ndarray],
                   budget: int = 1 << 27) -> np.ndarray:
    """int64 [n_q, n_pages]: the sign stage's S (include/b200ms.h, "sign candidates") of queries quantised to q8s (int
    [T_q, 128] each) over the sign rows uint8 [rows_padded, 16] of pages of `lens` true rows: +-1 rows times q8 in float64,
    where every product and partial sum is an integer of magnitude < 2^24, so exact."""
    device = sign_rows.device
    q8s = [np.asarray(q, dtype=np.int64).reshape(-1, 128) for q in q8s]
    q = torch.from_numpy(np.concatenate(q8s + [np.zeros((0, 128), np.int64)]).astype(np.float64)).to(device)
    out = _page_maxsim(q, lambda r0, r1: unpack_bits(sign_rows[r0:r1]).double() * 2 - 1, lens, [len(x) for x in q8s],
                       device, budget)
    return out.cpu().numpy().astype(np.int64)


def reference_scores(idx, q_packed: torch.Tensor, group_offsets, q_lens: Sequence[int],
                     device: Optional[torch.device] = None) -> np.ndarray:
    """reference_from_bytes on the bytes the scan of `idx` reads: idx.packed_rows() and the packed query block that
    score_groups returned with its group offsets.  Computed on `device` (default: the index's); float64 numpy result."""
    device = torch.device(device) if device is not None else idx.device
    rows = idx.packed_rows()
    if rows.device != device:
        rows = rows.to(device)
    q_u8 = q_packed.reshape(-1, idx.row_bytes)
    torch.cuda.synchronize(idx.device)
    return reference_from_bytes(idx.dtype_name, rows, idx.page_lens, q_u8.to(device), group_offsets, q_lens).cpu().numpy()


def token_maxima(dtype: str, rows_u8: torch.Tensor, row0: int, n: int, q_u8: torch.Tensor, group_offsets,
                 q_lens: Sequence[int]) -> List[np.ndarray]:
    """Per query, the float64 [T_q, n] token x row similarities (on the score scale) of one page of n true rows starting at
    padded row row0."""
    x = decode(dtype, rows_u8[row0:row0 + n]).to(q_u8.device)
    out = []
    for q, t in enumerate(q_lens):
        g0 = int(np.asarray(group_offsets)[q])
        sim = decode(dtype, q_u8[32 * g0:32 * g0 + int(t)]) @ x.T
        if dtype == "binary":
            sim = (sim + 128.0) / 2.0
        out.append((sim / _score_divisor(dtype)).cpu().numpy())
    return out
