"""oracle/maxsim_oracle.py -- TEST INFRASTRUCTURE ONLY.

CPU restatements of the reference's ColPali late-interaction path in numpy / torch-CPU, plus a ctypes
loader for the C restatement in ``maxsim_oracle.c``.  Only ``tests/``, ``__graft_entry__.smoke()`` and
``bench.py``'s ``cpu_baseline`` / ``--impl reference`` legs may import this module; the product package
(``morphik-core_b200/``) must never do so.

Reference lines restated (relative to the morphik-core repository root):
  * sign quantise + MSB-first pack : core/utils/fast_ops.py:191-227, morphik_rust/src/binary_ops.rs:147-222
  * Hamming                        : core/utils/fast_ops.py:230-248, morphik_rust/src/binary_ops.rs:237-292
  * binary MaxSim                  : core/vector_store/multi_vector_store.py:287-311 (SQL max_sim), :759 (ORDER BY)
  * float MaxSim                   : core/vector_store/fast_multivector_store.py:553-557 ->
                                     colpali_engine v0.3.13 ``score_multi_vector`` (third party; the identical port is
                                     transformers/models/colpali/processing_colpali.py:350-362)

Pinning status: quantiser/Hamming pinned by outputs of the reference's own ``fast_ops.py`` (tests/golden/
sign_pack.npz) and the Rust unit-test vectors; float MaxSim pinned by outputs of the transformers port of
``score_multi_vector`` (tests/golden/float_maxsim.npz); binary MaxSim pinned only by the known answers implied by
core/tests/unit/test_multivector.py (Postgres cannot run here); int8 MaxSim has no reference (SURVEY F5).
"""
from __future__ import annotations

import ctypes
import os
import subprocess
from typing import List, Optional, Sequence, Tuple

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
_LIB_PATH = os.path.join(_HERE, "_build", "liboracle.so")
_lib = None


def build_c_oracle(force: bool = False) -> str:
    """Compile maxsim_oracle.c (gcc) into oracle/_build/liboracle.so; returns the path."""
    srcs = [os.path.join(_HERE, f) for f in ("maxsim_oracle.c", "fde_oracle.c", "Makefile")]
    stale = (not os.path.exists(_LIB_PATH)) or any(os.path.getmtime(_LIB_PATH) < os.path.getmtime(f) for f in srcs)
    if force or stale:
        subprocess.run(["make", "-C", _HERE, "-s"] + (["-B"] if force else []), check=True)
    return _LIB_PATH


def c_oracle() -> ctypes.CDLL:
    global _lib
    if _lib is None:
        build_c_oracle()
        lib = ctypes.CDLL(_LIB_PATH)
        i64, i32, vp = ctypes.c_int64, ctypes.c_int, ctypes.c_void_p
        lib.oracle_max_threads.restype = i32
        lib.oracle_sign_pack.argtypes = [vp, i64, i32, vp]
        lib.oracle_hamming.argtypes = [vp, vp, i64]
        lib.oracle_hamming.restype = ctypes.c_uint32
        lib.oracle_binary_maxsim.argtypes = [vp, i32, vp, vp, i64, i32, vp, vp]
        lib.oracle_float_maxsim.argtypes = [vp, i32, vp, vp, i64, i32, i32, i32, vp]
        lib.oracle_int8_maxsim.argtypes = [vp, i32, vp, vp, i64, i32, i32, i32, vp]
        lib.oracle_topk.argtypes = [vp, i64, vp, i64, vp, vp]
        lib.oracle_topk.restype = i64
        lib.oracle_fde_encode.argtypes = [vp, i64, i32, i32, i32, i32, ctypes.c_float, vp, vp, vp, i32, vp]
        lib.oracle_fde_encode_ex.argtypes = [vp, i64, i32, i32, i32, i32, ctypes.c_float, vp, vp, vp, i32, i32, i32, vp, vp, vp]
        _lib = lib
    return _lib


def _ptr(a: Optional[np.ndarray]):
    return None if a is None else a.ctypes.data_as(ctypes.c_void_p)


def page_offsets(page_lens: Sequence[int]) -> np.ndarray:
    off = np.zeros(len(page_lens) + 1, dtype=np.int64)
    np.cumsum(np.asarray(page_lens, dtype=np.int64), out=off[1:])
    return off


# ------------------------------------------------------------------------------------------------
# numpy restatements (small sizes; these are what the C versions are cross-checked against)
# ------------------------------------------------------------------------------------------------
def sign_pack_np(x: np.ndarray) -> np.ndarray:
    """fast_ops.py:191-227: float32 cast, bit = x > 0, MSB-first pack -> uint8 [n, ceil(dim/8)]."""
    x = np.asarray(x)
    if x.dtype != np.float32:
        x = x.astype(np.float32)
    if x.ndim == 1:
        x = x[None, :]
    with np.errstate(invalid="ignore"):
        bits = x > 0
    return np.packbits(bits, axis=-1, bitorder="big")


def hamming_np(a: np.ndarray, b: np.ndarray) -> np.ndarray:
    """fast_ops.py:230-239: popcount(a XOR b) over the last axis of packed uint8 arrays."""
    return np.bitwise_count(np.bitwise_xor(a, b)).sum(axis=-1, dtype=np.int64)


def binary_maxsim_np(q_bits: np.ndarray, d_bits: np.ndarray, off: np.ndarray) -> Tuple[np.ndarray, np.ndarray]:
    """SQL max_sim (multi_vector_store.py:287-311).  Returns (float64 scores, exact int similarity)."""
    n_pages = len(off) - 1
    nbits = q_bits.shape[-1] * 8
    scores = np.zeros(n_pages, dtype=np.float64)
    sim_int = np.zeros(n_pages, dtype=np.int64)
    for p in range(n_pages):
        d = d_bits[off[p]:off[p + 1]]
        if d.shape[0] == 0 or q_bits.shape[0] == 0:
            continue  # COALESCE(SUM(...), 0.0)
        ham = hamming_np(q_bits[:, None, :], d[None, :, :])  # [T, P]
        sim = 1.0 - ham.astype(np.float64) / float(max(nbits, 1))
        scores[p] = sim.max(axis=1).sum()
        sim_int[p] = (nbits - ham.min(axis=1)).sum()
    return scores, sim_int


def float_maxsim_np(q: np.ndarray, rows: np.ndarray, off: np.ndarray, zero_pad_compat: bool = False,
                    batch: int = 128) -> np.ndarray:
    """score_multi_vector restated for one query (float64 accumulate, float32 out)."""
    n_pages = len(off) - 1
    lens = np.diff(off)
    out = np.zeros(n_pages, dtype=np.float32)
    q64 = q.astype(np.float64)
    for p in range(n_pages):
        d = rows[off[p]:off[p + 1]].astype(np.float64)
        padded = False
        if zero_pad_compat:
            b0 = (p // batch) * batch
            padded = lens[p] < lens[b0:b0 + batch].max()
        if d.shape[0] == 0 and not padded:
            continue
        sim = q64 @ d.T if d.shape[0] else np.zeros((q.shape[0], 0))
        best = sim.max(axis=1) if d.shape[0] else np.full(q.shape[0], -np.inf)
        if padded:
            best = np.maximum(best, 0.0)
        out[p] = np.float32(best.sum())
    return out


def int8_maxsim_np(q: np.ndarray, rows: np.ndarray, off: np.ndarray, zero_pad_compat: bool = False,
                   batch: int = 128) -> np.ndarray:
    """Integer MaxSim (int64 sums); zero_pad_compat / batch as in float_maxsim_np."""
    n_pages = len(off) - 1
    lens = np.diff(off)
    out = np.zeros(n_pages, dtype=np.int64)
    q32 = q.astype(np.int32)
    for p in range(n_pages):
        d = rows[off[p]:off[p + 1]].astype(np.int32)
        padded = False
        if zero_pad_compat:
            b0 = (p // batch) * batch
            padded = lens[p] < lens[b0:b0 + batch].max()
        if d.shape[0] == 0 and not padded:
            continue
        best = (q32 @ d.T).max(axis=1) if d.shape[0] else np.zeros(q.shape[0], dtype=np.int64)
        if padded:
            best = np.maximum(best, 0)
        out[p] = best.astype(np.int64).sum()
    return out


def rank_desc_np(scores: np.ndarray, ids: np.ndarray) -> np.ndarray:
    """Positions of `scores` in the build's order: score DESC, then id ASC.  Every NaN ranks above every number and NaNs
    tie with each other (torch.topk, Postgres ORDER BY ... DESC); -0.0 ties with +0.0."""
    with np.errstate(invalid="ignore"):
        s = np.asarray(scores).astype(np.float64) + 0.0  # -0.0 + 0.0 = +0.0
    nan = np.isnan(s)
    return np.lexsort((np.asarray(ids), -np.where(nan, 0.0, s), ~nan))


def topk_np(scores: np.ndarray, k: int, allow: Optional[np.ndarray] = None) -> Tuple[np.ndarray, np.ndarray]:
    """ORDER BY score DESC, page index ASC (the build's tie rule, rank_desc_np) LIMIT k; allow = bool mask per page."""
    ids = np.arange(len(scores), dtype=np.int64)
    if allow is not None:
        ids = ids[np.asarray(allow, dtype=bool)]
    s = np.asarray(scores)[ids]
    order = rank_desc_np(s, ids)[:k]
    return s[order], ids[order]


def quantize_int8_np(x: np.ndarray, scale: float) -> np.ndarray:
    """The build's int8 rule (no reference, SURVEY F5): round-half-even of the float32 product x * scale, clamped to
    [-127, 127] (so +-inf -> +-127); NaN -> 0 (it has neither sign nor magnitude)."""
    with np.errstate(over="ignore", invalid="ignore"):
        r = np.rint(np.asarray(x, dtype=np.float32) * np.float32(scale))
    return np.where(np.isnan(r), 0, np.clip(r, -127, 127)).astype(np.int8)


def bf16_round_np(x: np.ndarray) -> np.ndarray:
    """fp32 -> bf16 (round-to-nearest-even; overflow -> +-inf; subnormals kept) -> fp32, bit-exact with the device's
    cvt.rn.bf16x2.f32: every NaN becomes the canonical bf16 NaN 0x7fff (sign dropped; torch's own cast writes 0x7fc0)."""
    u = np.asarray(x, dtype=np.float32).view(np.uint32).astype(np.uint64)
    rounded = ((u + 0x7FFF + ((u >> 16) & 1)) >> 16) << 16
    nan = (u & 0x7FFFFFFF) > 0x7F800000
    return np.where(nan, np.uint64(0x7FFF0000), rounded).astype(np.uint32).view(np.float32)


# ------------------------------------------------------------------------------------------------
# C-backed versions (fast; used at the sizes the GPU parity tests and the CPU baseline need)
# ------------------------------------------------------------------------------------------------
def sign_pack_c(x: np.ndarray) -> np.ndarray:
    x = np.ascontiguousarray(x, dtype=np.float32)
    if x.ndim == 1:
        x = x[None, :]
    n, dim = x.shape
    out = np.empty((n, (dim + 7) // 8), dtype=np.uint8)
    c_oracle().oracle_sign_pack(_ptr(x), n, dim, _ptr(out))
    return out


def binary_maxsim_c(q_bits: np.ndarray, d_bits: np.ndarray, off: np.ndarray) -> Tuple[np.ndarray, np.ndarray]:
    q_bits = np.ascontiguousarray(q_bits, dtype=np.uint8)
    d_bits = np.ascontiguousarray(d_bits, dtype=np.uint8)
    off = np.ascontiguousarray(off, dtype=np.int64)
    n_pages = len(off) - 1
    scores = np.zeros(n_pages, dtype=np.float64)
    sim_int = np.zeros(n_pages, dtype=np.int64)
    c_oracle().oracle_binary_maxsim(_ptr(q_bits), q_bits.shape[0], _ptr(d_bits), _ptr(off), n_pages,
                                    q_bits.shape[1], _ptr(scores), _ptr(sim_int))
    return scores, sim_int


def float_maxsim_c(q: np.ndarray, rows: np.ndarray, off: np.ndarray, zero_pad_compat: bool = False,
                   batch: int = 128) -> np.ndarray:
    q = np.ascontiguousarray(q, dtype=np.float32)
    rows = np.ascontiguousarray(rows, dtype=np.float32)
    off = np.ascontiguousarray(off, dtype=np.int64)
    n_pages = len(off) - 1
    out = np.zeros(n_pages, dtype=np.float32)
    c_oracle().oracle_float_maxsim(_ptr(q), q.shape[0], _ptr(rows), _ptr(off), n_pages, q.shape[1],
                                   int(zero_pad_compat), batch, _ptr(out))
    return out


def int8_maxsim_c(q: np.ndarray, rows: np.ndarray, off: np.ndarray, zero_pad_compat: bool = False,
                  batch: int = 128) -> np.ndarray:
    q = np.ascontiguousarray(q, dtype=np.int8)
    rows = np.ascontiguousarray(rows, dtype=np.int8)
    off = np.ascontiguousarray(off, dtype=np.int64)
    n_pages = len(off) - 1
    out = np.zeros(n_pages, dtype=np.int64)
    c_oracle().oracle_int8_maxsim(_ptr(q), q.shape[0], _ptr(rows), _ptr(off), n_pages, q.shape[1],
                                  int(zero_pad_compat), batch, _ptr(out))
    return out


def topk_c(scores: np.ndarray, k: int, allow_bits: Optional[np.ndarray] = None) -> Tuple[np.ndarray, np.ndarray]:
    s = np.ascontiguousarray(scores, dtype=np.float64)
    ts = np.zeros(k, dtype=np.float64)
    ti = np.zeros(k, dtype=np.int64)
    if allow_bits is not None:
        allow_bits = np.ascontiguousarray(allow_bits, dtype=np.uint32)
    n = c_oracle().oracle_topk(_ptr(s), len(s), _ptr(allow_bits), k, _ptr(ts), _ptr(ti))
    return ts[:n], ti[:n]


# ------------------------------------------------------------------------------------------------
# The reference's own formulation, executed on the host CPU (used as the `--impl reference` arm):
# colpali_engine v0.3.13 score_multi_vector == pad_sequence + einsum("bnd,csd->bcns").max(3).sum(2)
# ------------------------------------------------------------------------------------------------
def score_multi_vector_port(qs: List["np.ndarray"], ps: List["np.ndarray"], batch_size: int = 128):
    """Restates fast_multivector_store.py:553-555's callee with torch on CPU (fp32, all host threads).

    qs: list of [T_i, D] arrays, ps: list of [P_j, D] arrays -> float32 [len(qs), len(ps)] (torch tensor).
    """
    import torch

    tq = [torch.as_tensor(np.asarray(q, dtype=np.float32)) for q in qs]
    tp = [torch.as_tensor(np.asarray(p, dtype=np.float32)) for p in ps]
    scores = []
    for i in range(0, len(tq), batch_size):
        qb = torch.nn.utils.rnn.pad_sequence(tq[i:i + batch_size], batch_first=True, padding_value=0)
        row = []
        for j in range(0, len(tp), batch_size):
            pb = torch.nn.utils.rnn.pad_sequence(tp[j:j + batch_size], batch_first=True, padding_value=0)
            row.append(torch.einsum("bnd,csd->bcns", qb, pb).max(dim=3)[0].sum(dim=2))
        scores.append(torch.cat(row, dim=1).to(torch.float32))
    return torch.cat(scores, dim=0)


def score_multi_vector_port_dense(q: "np.ndarray", p: "np.ndarray", batch_size: int = 128):
    """Same arithmetic for already-dense inputs q [B,T,D], p [C,P,D] (equal-length pages: no padding needed)."""
    import torch

    tq = torch.as_tensor(np.asarray(q, dtype=np.float32))
    tp = torch.as_tensor(np.asarray(p, dtype=np.float32))
    out = []
    for i in range(0, tq.shape[0], batch_size):
        row = []
        for j in range(0, tp.shape[0], batch_size):
            row.append(torch.einsum("bnd,csd->bcns", tq[i:i + batch_size], tp[j:j + batch_size]).max(dim=3)[0].sum(dim=2))
        out.append(torch.cat(row, dim=1))
    return torch.cat(out, dim=0)


# ------------------------------------------------------------------------------------------------
# FDE (MUVERA) -- parity unpinned (sources absent from the reference, SURVEY F2); see oracle/fde_oracle.c
# ------------------------------------------------------------------------------------------------
def fde_encode_c(x: np.ndarray, simhash: np.ndarray, ams_index: np.ndarray, ams_sign: np.ndarray, scale: float,
                 is_document: bool) -> np.ndarray:
    """x [n,128] float32 -> FDE float32 [reps * 2^ksim * proj] with the loop order the device kernel uses."""
    x = np.ascontiguousarray(x, dtype=np.float32)
    simhash = np.ascontiguousarray(simhash, dtype=np.float32)
    ams_index = np.ascontiguousarray(ams_index, dtype=np.int32)
    ams_sign = np.ascontiguousarray(ams_sign, dtype=np.float32)
    reps, dim, ksim = simhash.shape
    proj = int(ams_index.max()) + 1 if ams_index.size else 1
    return fde_encode_c_proj(x, simhash, ams_index, ams_sign, scale, is_document, proj)


def fde_encode_c_proj(x, simhash, ams_index, ams_sign, scale, is_document, proj) -> np.ndarray:
    reps, dim, ksim = simhash.shape
    out = np.zeros(reps * (1 << ksim) * proj, dtype=np.float32)
    c_oracle().oracle_fde_encode(_ptr(x), x.shape[0], dim, reps, ksim, proj, ctypes.c_float(scale), _ptr(simhash),
                                 _ptr(ams_index), _ptr(ams_sign), int(is_document), _ptr(out))
    return out


def fde_encode_c_ex(x, simhash, ams_index, ams_sign, scale, is_document, proj, fill_empty=False, final_index=None,
                    final_sign=None, final_dim=0) -> np.ndarray:
    """oracle_fde_encode_ex: + fill_empty_partitions and the final count-sketch projection."""
    x = np.ascontiguousarray(x, dtype=np.float32)
    simhash = np.ascontiguousarray(simhash, dtype=np.float32)
    ams_index = np.ascontiguousarray(ams_index, dtype=np.int32)
    ams_sign = np.ascontiguousarray(ams_sign, dtype=np.float32)
    reps, dim, ksim = simhash.shape
    inner = reps * (1 << ksim) * proj
    out = np.zeros(final_dim if final_dim > 0 else inner, dtype=np.float32)
    fi = None if final_dim <= 0 else np.ascontiguousarray(final_index, dtype=np.int32)
    fs = None if final_dim <= 0 else np.ascontiguousarray(final_sign, dtype=np.float32)
    c_oracle().oracle_fde_encode_ex(_ptr(x), x.shape[0], dim, reps, ksim, proj, ctypes.c_float(scale), _ptr(simhash),
                                    _ptr(ams_index), _ptr(ams_sign), int(is_document), int(fill_empty), int(final_dim),
                                    _ptr(fi), _ptr(fs), _ptr(out))
    return out


# ------------------------------------------------------------------------------------------------
# fp8 e4m3 (B200MS_F8 corpora; new relative to the reference, like int8): round-to-nearest-even onto the 127 finite
# non-negative e4m3 values, saturating at 448 -- what __nv_cvt_float_to_fp8(x, __NV_SATFINITE, __NV_E4M3) does.
# ------------------------------------------------------------------------------------------------
def _e4m3_table() -> np.ndarray:
    vals = []
    for code in range(0x7F):  # 0x7f is NaN
        e, m = code >> 3, code & 7
        vals.append((m / 8.0) * 2.0 ** -6 if e == 0 else (1.0 + m / 8.0) * 2.0 ** (e - 7))
    return np.asarray(vals, dtype=np.float64)


_E4M3 = _e4m3_table()


def quantize_e4m3_np(x: np.ndarray, scale: float = 64.0) -> np.ndarray:
    """float -> e4m3 CODES (uint8) of the float32 product x*scale (the library multiplies in fp32, then rounds once more):
    round-to-nearest-even (ties -> even code), |x*scale| > 448 and +-inf saturate to +-448, NaN -> 0x7f (sign dropped)."""
    with np.errstate(over="ignore", invalid="ignore"):
        y32 = np.asarray(x, dtype=np.float32) * np.float32(scale)
    y = y32.astype(np.float64)
    nan = np.isnan(y)
    a = np.minimum(np.abs(np.where(nan, 0.0, y)), 448.0)
    hi = np.clip(np.searchsorted(_E4M3, a, side="left"), 0, len(_E4M3) - 1)
    lo = np.maximum(hi - 1, 0)
    d_lo, d_hi = a - _E4M3[lo], _E4M3[hi] - a
    pick_hi = (d_hi < d_lo) | ((d_hi == d_lo) & (hi % 2 == 0))
    code = np.where(pick_hi, hi, lo).astype(np.uint8) | (np.signbit(y32).astype(np.uint8) << 7)
    return np.where(nan, np.uint8(0x7F), code).astype(np.uint8)


def dequantize_e4m3_np(codes: np.ndarray) -> np.ndarray:
    c = np.asarray(codes, dtype=np.uint8)
    v = _E4M3[(c & 0x7F).astype(np.int64)]
    return np.where(c & 0x80, -v, v).astype(np.float32)


def fde_encode_np(x: np.ndarray, simhash: np.ndarray, ams_index: np.ndarray, ams_sign: np.ndarray, scale: float,
                  is_document: bool, proj: int, fill_empty: bool = False, final_index: Optional[np.ndarray] = None,
                  final_sign: Optional[np.ndarray] = None, final_dim: int = 0) -> np.ndarray:
    """Independent numpy restatement (float64 arithmetic) used to cross-check the C loops within rounding.

    A row whose SimHash dot lies near zero may fall into another partition here than in the fp32 loops; callers draw rows
    with a margin so that the partitions agree."""
    x = np.asarray(x, dtype=np.float64)
    reps, dim, ksim = simhash.shape
    n_part = 1 << ksim
    out = np.zeros((reps, n_part, proj))
    for r in range(reps):
        bits = (x @ simhash[r].astype(np.float64)) > 0  # [n, ksim]
        code = np.zeros(x.shape[0], dtype=np.int64)
        sign_bits = np.zeros(x.shape[0], dtype=np.int64)  # first projection in the most significant bit
        for k in range(ksim):
            code = (code << 1) + (bits[:, k].astype(np.int64) ^ (code & 1))
            sign_bits = (sign_bits << 1) | bits[:, k].astype(np.int64)
        A = np.zeros((dim, proj))
        A[np.arange(dim), ams_index[r]] = ams_sign[r]
        y = x @ A
        for p in range(n_part):
            sel = code == p
            if sel.any():
                out[r, p] = y[sel].sum(axis=0) * scale / (sel.sum() if is_document else 1.0)
            elif is_document and fill_empty and x.shape[0]:
                # partition p holds the rows whose sign bits are p's Gray code; nearest by Hamming distance, first wins
                dist = np.bitwise_count(sign_bits ^ (p ^ (p >> 1)))
                out[r, p] = y[int(np.argmin(dist))] * scale
    v = out.reshape(-1)
    if final_dim > 0:
        f = np.zeros(final_dim)
        np.add.at(f, np.asarray(final_index, dtype=np.int64), np.asarray(final_sign, dtype=np.float64) * v)
        v = f
    return v.astype(np.float32)
