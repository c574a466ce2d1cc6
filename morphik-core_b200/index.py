"""MaxSimIndex -- a device-resident, packed multi-vector corpus plus the search calls over it.

This is the piece that replaces the reference's exhaustive scorers:
  * Postgres evaluating SQL ``max_sim`` over every ``multi_vector_embeddings`` row
    (core/vector_store/multi_vector_store.py:287-311, 746-763)            -> dtype "binary"
  * ``ColQwen2_5_Processor.score_multi_vector`` + ``torch.topk``
    (core/vector_store/fast_multivector_store.py:553-557)                -> dtype "bf16"
  * (new, BASELINE config 3) integer MaxSim over int8 patches            -> dtype "int8"

PyTorch is used only to own device memory and to name the current stream; every computation goes through the
C-ABI of libb200ms.so (``_native``).  Nothing here falls back to the CPU.
"""
from __future__ import annotations

import ctypes
import math
from typing import List, Optional, Sequence, Tuple, Union

import numpy as np
import torch

from . import _native as nat
from .catalog import PageCatalog

ArrayLike = Union[np.ndarray, torch.Tensor]


def _vp(t: Optional[torch.Tensor]):
    return None if t is None else ctypes.c_void_p(t.data_ptr())


# sources per first-stage call of a duplicate-candidate search: bounds the query rows staged at once (a 1030-row source
# is 1030 query tokens)
DUP_SOURCE_BATCH = 64


def _check_n_candidates(n_candidates) -> int:
    n = int(n_candidates)
    if n < 1:
        raise ValueError(f"n_candidates must be >= 1, got {n_candidates}")
    return n


def candidate_pairs(parts, n_candidates: int, device) -> Tuple[torch.Tensor, torch.Tensor]:
    """Candidate lists -> canonical page pairs.  parts: (source ids, device int64 [n_src, width] candidate ids, -1 =
    unused) per batch; each source keeps its first n_candidates candidates other than itself.  Returns device int64
    (pair_a, pair_b) with pair_a < pair_b, unique, ordered by (a, b)."""
    lo, hi = [], []
    for src, ti in parts:
        s = torch.as_tensor(src, dtype=torch.int64, device=ti.device).view(-1, 1).expand_as(ti)
        ok = (ti >= 0) & (ti != s)
        ok &= torch.cumsum(ok.to(torch.int32), dim=1) <= int(n_candidates)
        a, b = s[ok], ti[ok]
        lo.append(torch.minimum(a, b))
        hi.append(torch.maximum(a, b))
    if not lo:
        empty = torch.zeros((0,), dtype=torch.int64, device=device)
        return empty, empty.clone()
    lo_t, hi_t = torch.cat(lo), torch.cat(hi)
    base = int(hi_t.max().item()) + 1 if hi_t.numel() else 1
    key = torch.unique(lo_t * base + hi_t, sorted=True)
    return (key // base).contiguous(), (key % base).contiguous()


def _aligned_bytes(nbytes: int, device: torch.device, align: int = 1024) -> torch.Tensor:
    """uint8 device tensor whose data_ptr is `align`-byte aligned (set_corpus / TMA want 1024)."""
    raw = torch.empty(max(int(nbytes), 1) + align, dtype=torch.uint8, device=device)
    off = (-raw.data_ptr()) % align
    return raw[off:off + max(int(nbytes), 1)]


def _padded_lens(lens: Sequence[int]) -> np.ndarray:
    """int64 rows each page occupies in the packed layout: its length rounded up to whole 32-row groups
    (= b200ms_padded_len, computed here for every page at once)."""
    return -(-np.asarray(lens, dtype=np.int64) // nat.ROW_GROUP) * nat.ROW_GROUP


def _runs(ids: Sequence[int]):
    """(first, last) of every maximal run of consecutive ids in ascending `ids`."""
    i = 0
    while i < len(ids):
        j = i
        while j + 1 < len(ids) and ids[j + 1] == ids[j] + 1:
            j += 1
        yield ids[i], ids[j]
        i = j + 1


def _row_runs(page_lens: Sequence[int], keep: Sequence[int]) -> List[Tuple[int, int]]:
    """Packed row ranges [a, b) of the maximal runs of consecutive pages in ascending `keep`."""
    starts = np.concatenate([[0], np.cumsum(_padded_lens(page_lens))]).astype(np.int64)
    return [(int(starts[first]), int(starts[last + 1])) for first, last in _runs(keep)]


# ---- argument checks of the device calls: tensor metadata only (no value is read, nothing synchronises or is allocated),
# so a tensor the library would read past its end or in the wrong format is refused with ValueError before any launch
def _check_queries(q_dev: torch.Tensor, q_lens: Sequence[int], device: torch.device) -> int:
    """Query rows: contiguous float32/bfloat16 [>= sum(q_lens), 128] on `device`.  Returns the library's dtype code."""
    if q_dev.dtype not in (torch.float32, torch.bfloat16) or not q_dev.is_contiguous() or q_dev.device != device:
        raise ValueError(f"q_dev must be a contiguous float32/bfloat16 tensor on {device}, got {q_dev.dtype} on {q_dev.device}")
    rows = sum(int(n) for n in q_lens)
    if q_dev.ndim != 2 or q_dev.shape[1] != nat.DIM or q_dev.shape[0] < rows:
        raise ValueError(f"q_dev must be [>= sum(q_lens) = {rows}, {nat.DIM}], got {tuple(q_dev.shape)}")
    return nat.BF16 if q_dev.dtype == torch.bfloat16 else nat.F32


def _check_device_masks(allow_mask_dev: Optional[torch.Tensor], mask_index_dev: Optional[torch.Tensor], n_q: int,
                        n_pages: int, device: torch.device):
    """Allow filter on `device`, int32/uint32 words (bit p&31 of word p>>5): one [ceil(n_pages/32)] row for every query, or a
    [n_masks, ceil(n_pages/32)] matrix with ``mask_index_dev`` int32 [n_q] naming each query's row (-1 = unfiltered).
    Returns (masks, n_masks, index) for the C call: (None, 0, None) unfiltered, (row, 1, None) for one row."""
    words = (n_pages + 31) // 32
    if allow_mask_dev is None:
        if mask_index_dev is not None:
            raise ValueError("mask_index_dev needs allow_mask_dev")
        return None, 0, None
    m = allow_mask_dev
    if m.dtype not in (torch.int32, torch.uint32) or not m.is_contiguous() or m.device != device:
        raise ValueError(f"allow_mask_dev must be a contiguous int32/uint32 tensor on {device}, got {m.dtype} on {m.device}")
    if mask_index_dev is None:
        if tuple(m.shape) != (words,):
            raise ValueError(f"allow_mask_dev must have {words} words for {n_pages} pages, got shape {tuple(m.shape)}")
        return m, 1, None
    if m.ndim != 2 or m.shape[1] != words:
        raise ValueError(f"per-query masks: allow_mask_dev must be a [n_masks, {words}] word matrix, got {tuple(m.shape)}")
    mi = mask_index_dev
    if mi.dtype != torch.int32 or tuple(mi.shape) != (n_q,) or not mi.is_contiguous() or mi.device != device:
        raise ValueError(f"mask_index_dev must be a contiguous int32 [{n_q}] tensor on {device}")
    return m, int(m.shape[0]), mi


def _host_mask_words(allow_mask, n_pages: int) -> np.ndarray:
    """Host allow mask -> contiguous uint32 words.  The library reads ceil(n_pages/32) words: a mask built for an older
    (shorter) corpus must never reach it."""
    m = np.ascontiguousarray(allow_mask, dtype=np.uint32)
    words = (n_pages + 31) // 32
    if m.shape != (words,):
        raise ValueError(f"allow-mask must have {words} uint32 words for {n_pages} pages, got shape {m.shape}")
    return m


def _host_mask_to_device(allow_mask: Optional[np.ndarray], n_pages: int, device: torch.device) -> Optional[torch.Tensor]:
    """Checked host allow mask (uint32 words) -> int32 words on `device`; None stays None (unfiltered)."""
    if allow_mask is None:
        return None
    return torch.from_numpy(_host_mask_words(allow_mask, n_pages).view(np.int32)).to(device)


def _check_candidates(cand_ids: torch.Tensor, n_q: int, k: int, device: torch.device, per_query: bool) -> Tuple[int, int]:
    """Candidate page ids: contiguous int64 [n_cand] shared by every query, or with ``per_query`` [n_q, n_cand], on `device`.
    Returns (n_cand, k capped at n_cand)."""
    shape = "[n_q, n_cand]" if per_query else "[n_cand]"
    ok_shape = cand_ids.ndim == 2 and cand_ids.shape[0] == n_q if per_query else cand_ids.ndim == 1
    if cand_ids.dtype != torch.int64 or not ok_shape or not cand_ids.is_contiguous() or cand_ids.device != device:
        raise ValueError(f"cand_ids must be a contiguous int64 {shape} tensor on {device} (n_q = {n_q}), "
                         f"got {cand_ids.dtype} {tuple(cand_ids.shape)} on {cand_ids.device}")
    n_cand = int(cand_ids.shape[-1])
    return n_cand, int(min(k, n_cand))


def _topk_outputs(n_q: int, k: int, device: torch.device, out=None, per_doc: int = 0):
    """Result buffers of a top-k call on `device`: (scores float32 [n_q,k], page ids int64 [n_q,k], counts int32 [n_q]), or
    with ``per_doc`` the grouped form (scores float32 [n_q,k,per_doc], page ids int64 [n_q,k,per_doc], pages per document
    int32 [n_q,k], documents int32 [n_q]).  Allocated when `out` is None, else the caller's tuple is checked to be exactly
    that and returned."""
    row = (n_q, k, per_doc) if per_doc else (n_q, k)
    specs = [(row, torch.float32), (row, torch.int64)] + ([((n_q, k), torch.int32)] if per_doc else []) + [((n_q,), torch.int32)]
    if out is None:
        return tuple(torch.empty(shape, dtype=dt, device=device) for shape, dt in specs)
    if len(out) != len(specs) or any(tuple(t.shape) != shape or t.dtype != dt or not t.is_contiguous() or t.device != device
                                     for t, (shape, dt) in zip(out, specs)):
        want = ", ".join(f"{str(dt).replace('torch.', '')} {list(shape)}" for shape, dt in specs)
        raise ValueError(f"out must be contiguous tensors on {device}: {want}")
    return tuple(out)


class HostBlock:
    """Pinned, device-mapped host memory of exactly ``nbytes`` (b200ms_host_alloc), freed by ``free`` or garbage collection.

    torch's pinned allocator rounds requests up to a power of two, which would turn a 262 GB corpus into a 512 GB
    reservation; this block is sized exactly.  ``tensor`` is a CPU uint8 view of it: views taken from it must not outlive
    the block."""

    def __init__(self, handle: "nat.Handle", nbytes: int):
        p = ctypes.c_void_p()
        handle.check(nat.lib.b200ms_host_alloc(handle.ptr, int(nbytes), ctypes.byref(p)), "b200ms_host_alloc")
        self.handle, self.ptr, self.nbytes = handle, int(p.value), int(nbytes)
        arr = np.ctypeslib.as_array((ctypes.c_uint8 * max(self.nbytes, 1)).from_address(self.ptr))
        self.tensor = torch.from_numpy(arr)

    def free(self):
        if self.ptr:
            self.tensor = None
            nat.lib.b200ms_host_free(self.handle.ptr, ctypes.c_void_p(self.ptr))
            self.ptr = 0

    def __del__(self):
        try:
            self.free()
        except Exception:
            pass


class _CudaBytes:
    """`nbytes` device bytes at `ptr` as an object torch.as_tensor accepts; it owns nothing."""

    def __init__(self, ptr: int, nbytes: int):
        self.__cuda_array_interface__ = {"shape": (int(nbytes),), "typestr": "|u1", "data": (int(ptr), False), "version": 2}


class DeviceBlock:
    """Growable HBM block (b200ms_block_*): address space for the whole card is reserved once, and ``resize`` backs exactly
    as much of it as asked (in chunks of 32 MiB), so a corpus grows without a copy or a second buffer and shrinks by handing
    memory back to the driver; the address never changes.  The memory lives outside torch's allocator.

    ``tensor`` is a uint8 device view of the backed bytes (None while nothing is backed), made anew by every ``resize``:
    views taken from it must not outlive the block, nor a shrink that cuts them off."""

    def __init__(self, handle: "nat.Handle", device: torch.device):
        p = ctypes.c_void_p()
        total = torch.cuda.get_device_properties(device).total_memory
        handle.check(nat.lib.b200ms_block_create(handle.ptr, int(total), ctypes.byref(p)), "b200ms_block_create")
        self.handle, self.device, self.ptr = handle, device, p
        self.tensor: Optional[torch.Tensor] = None

    def resize(self, nbytes: int):
        self.tensor = None
        try:
            self.handle.check(nat.lib.b200ms_block_resize(self.handle.ptr, self.ptr, int(nbytes)), "b200ms_block_resize")
        finally:  # a refused resize leaves the block as it was
            mapped = int(nat.lib.b200ms_block_mapped_bytes(self.ptr))
            if mapped:
                self.tensor = torch.as_tensor(_CudaBytes(nat.lib.b200ms_block_ptr(self.ptr), mapped), device=self.device)

    @staticmethod
    def resized(block: Optional["DeviceBlock"], handle: "nat.Handle", device: torch.device, nbytes: int) -> "DeviceBlock":
        """`block` -- or, when None, a new block -- backing `nbytes`; a new block whose resize is refused is freed again."""
        new = DeviceBlock(handle, device) if block is None else block
        try:
            new.resize(nbytes)
        except Exception:
            if block is None:
                new.free()
            raise
        return new

    def rows(self, row_bytes: int) -> Optional[torch.Tensor]:
        """The backed bytes as whole rows: uint8 [backed // row_bytes, row_bytes], None while nothing is backed."""
        if self.tensor is None:
            return None
        n = self.tensor.numel() // row_bytes
        return self.tensor[: n * row_bytes].view(n, row_bytes)

    def free(self):
        self.tensor = None
        if self.ptr and self.handle.ptr:  # a closed handle has released its blocks already
            nat.lib.b200ms_block_destroy(self.handle.ptr, self.ptr)
        self.ptr = None

    def __del__(self):
        try:
            self.free()
        except Exception:
            pass


def _compact_rows(h: "nat.Handle", device: torch.device, rows: torch.Tensor, row_bytes: int,
                  runs: Sequence[Tuple[int, int]]) -> None:
    """Move the row ranges [a, b) of `runs` (ascending) down to the front of `rows`, in place on the GPU, with one
    b200ms_compact_rows call.  Returns once torch's stream is idle: the block's shrink that follows unmaps the freed tail
    after the handle's calls, but copies torch itself queued on those rows (append_packed, the FDE rows' copies) are only
    known to this stream."""
    run_start = np.array([a for a, _ in runs], dtype=np.int64)
    run_rows = np.array([b - a for a, b in runs], dtype=np.int64)
    stream = ctypes.c_void_p(torch.cuda.current_stream(device).cuda_stream)
    with torch.cuda.device(device):
        h.check(nat.lib.b200ms_compact_rows(h.ptr, _vp(rows), row_bytes, run_start.ctypes.data_as(nat.i64p),
                                            run_rows.ctypes.data_as(nat.i64p), len(runs), stream),
                "b200ms_compact_rows")
    torch.cuda.current_stream(device).synchronize()


class MaxSimIndex:
    """Packed corpus of pages (each a [P_i, 128] matrix of patch embeddings) on one GPU.

    Layout in HBM: rows of ``row_bytes`` (bf16 256 B / int8 128 B / sign bits 16 B), every page padded to a
    multiple of 32 rows by repeating its last row, pages back to back in insertion order.  ``page id`` = insertion index.

    ``tier="host"`` keeps the same packed rows in pinned host memory (``HostBlock``) instead of HBM, so the corpus is bounded
    by host RAM rather than by the card: only ``rerank`` / ``rerank_batch`` work on it (each call copies just its candidate
    pages over PCIe into an HBM staging block, with scores bit-identical to the HBM tier); the ``search_*`` full scans
    raise ``NativeError``.  Growing the block allocates a new one and copies, so it briefly needs twice the corpus in
    pinned memory; ``capacity_rows`` sizes the block once up front and avoids that.

    ``tier="hbm"`` keeps the rows in a ``DeviceBlock``: growing backs more of the block (no copy, no second buffer),
    ``compact`` moves the surviving rows down in place and returns the freed tail to the driver, so a corpus that is
    ingested into and deleted from can fill the card.  ``capacity_rows`` / ``reserve_rows`` only back the memory early.
    """

    def __init__(self, device: int = 0, dtype: str = "bf16", i8_scale: float = 127.0, capacity_rows: int = 0,
                 tier: str = "hbm"):
        if dtype not in nat.DTYPE_NAMES or nat.DTYPE_NAMES[dtype] == nat.F32:
            raise ValueError(f"dtype must be one of bf16/int8/fp8/binary, got {dtype!r}")
        if tier not in ("hbm", "host"):
            raise ValueError(f"tier must be 'hbm' or 'host', got {tier!r}")
        if not torch.cuda.is_available():
            raise nat.NativeError("MaxSimIndex needs a CUDA device (H100); there is no CPU fallback")
        self.tier = tier
        # owner of the memory self._buf views: a HostBlock (host tier) or a DeviceBlock; None while an HBM index is empty
        # or uses a caller's tensor (adopt_packed)
        self._block: Union[HostBlock, DeviceBlock, None] = None
        self.device = torch.device("cuda", int(device))
        self.dtype = nat.DTYPE_NAMES[dtype]
        self.dtype_name = dtype
        self.row_bytes = nat.ROW_BYTES[self.dtype]
        # corpus AND query quantisation scale: int8 rint(x*127) for unit-norm rows; fp8 e4m3(x*64) -- a power of two keeps the
        # scaling exact and puts |x| in [2^-12, 7] into e4m3's normal range
        self.i8_scale = 64.0 if (self.dtype == nat.F8 and float(i8_scale) == 127.0) else float(i8_scale)
        self.h = nat.Handle(int(device))
        self._buf: Optional[torch.Tensor] = None  # aligned uint8 storage of the packed rows
        self._cap_rows = 0
        self._rows = 0  # padded rows in use
        self._page_lens: List[int] = []
        self._attached = False
        if capacity_rows:
            self._grow(int(capacity_rows))

    # ------------------------------------------------------------------ properties
    @property
    def n_pages(self) -> int:
        return len(self._page_lens)

    @property
    def n_rows_padded(self) -> int:
        return self._rows

    @property
    def page_lens(self) -> np.ndarray:
        return np.asarray(self._page_lens, dtype=np.int32)

    @property
    def score_scale(self) -> float:
        """Factor that turns the kernels' raw sums into reference-scale scores."""
        if self.dtype == nat.B1:
            return 1.0 / 128.0  # sum_t max_r (128 - ham) / 128  == SQL max_sim
        if self.dtype in (nat.I8, nat.F8):
            return 1.0 / (self.i8_scale * self.i8_scale)
        return 1.0

    @property
    def float_scores(self) -> bool:
        """True when the kernels emit float32 group scores (bf16 / fp8 corpora), False for exact int32 (int8 / binary)."""
        return self.dtype in (nat.BF16, nat.F8)

    def launch_count(self) -> int:
        return int(nat.lib.b200ms_launch_count(self.h.ptr))

    def last_score_ms(self) -> float:
        ms = float(nat.lib.b200ms_last_score_ms(self.h.ptr))
        if ms < 0:
            self.h.check(int(ms), "b200ms_last_score_ms")
        return ms

    def score_times_ms(self, n: int) -> List[float]:
        """Device times (ms) of the scoring kernels of the last n score/search calls (CUDA events on the launch stream)."""
        buf = (ctypes.c_float * max(n, 1))()
        rc = nat.lib.b200ms_score_times_ms(self.h.ptr, buf, int(n))
        if rc < 0:
            self.h.check(rc, "b200ms_score_times_ms")
        return [float(buf[i]) for i in range(n)]

    def set_tuning(self, unit_rows: int = 0, max_ctas: int = 0):
        self.h.check(nat.lib.b200ms_set_tuning(self.h.ptr, int(unit_rows), int(max_ctas)), "b200ms_set_tuning")
        self._attached = False

    def set_option(self, name: str, value: int):
        self.h.check(nat.lib.b200ms_set_option(self.h.ptr, name.encode(), int(value)), f"b200ms_set_option({name})")
        if name == "unit_rows":
            self._attached = False

    def _stream(self):
        return ctypes.c_void_p(torch.cuda.current_stream(self.device).cuda_stream)

    # ------------------------------------------------------------------ building the corpus
    def _grow(self, need_rows: int, exact: bool = False):
        if need_rows <= self._cap_rows:
            return
        if self.tier == "hbm":
            self._resize_block(need_rows)
            return
        new_cap = need_rows if exact else max(need_rows, int(self._cap_rows * 1.5), 4096)
        self._host_barrier()
        block = HostBlock(self.h, new_cap * self.row_bytes)
        new_buf = block.tensor
        if self._buf is not None and self._rows:
            new_buf[: self._rows * self.row_bytes].copy_(self._buf[: self._rows * self.row_bytes])
        if self._block is not None:
            self._buf = None
            self._block.free()
        self._block = block
        self._buf = new_buf
        self._cap_rows = new_cap
        self._attached = False

    def _resize_block(self, rows: int):
        """HBM tier: back exactly `rows` rows (rounded up to whole chunks) of the index's block; the rows that stay keep
        their contents and address.  Rows held in a caller's tensor (``adopt_packed``) move into a block of their own
        first, which is the one copy such a corpus ever makes."""
        block = DeviceBlock.resized(self._block, self.h, self.device, rows * self.row_bytes)
        if self._block is None and self._buf is not None and self._rows:
            block.tensor[: self._rows * self.row_bytes].copy_(self._buf[: self._rows * self.row_bytes])
        self._block, self._buf = block, block.tensor
        self._cap_rows = 0 if self._buf is None else self._buf.numel() // self.row_bytes
        self._attached = False

    def reserve_rows(self, rows: int):
        """Make room for `rows` padded rows in total with one allocation of exactly that size (host tier: avoids the
        transient second copy that growth needs; HBM tier: backs the block's memory now instead of as the pages arrive)."""
        self._grow(int(rows), exact=True)

    def _host_barrier(self):
        """A rerank of the host tier still queued on some stream may read the block: wait for the device before any host
        write to it."""
        if self.tier == "host" and self._block is not None:
            torch.cuda.synchronize(self.device)

    def tail(self, nbytes: int) -> torch.Tensor:
        """Writable uint8 view of the `nbytes` just past the used rows, grown to fit: of the pinned block on the host tier
        (a CPU tensor), of the device block on the HBM tier.  ``commit_rows`` appends the packed pages written into it."""
        nbytes = int(nbytes)
        self._grow(self._rows + -(-nbytes // self.row_bytes))
        self._host_barrier()
        if self._buf is None:  # nothing backed and nothing asked for
            return torch.empty(0, dtype=torch.uint8, device=self.device if self.tier == "hbm" else "cpu")
        o = self._rows * self.row_bytes
        return self._buf[o:o + nbytes]

    def commit_rows(self, page_lens: Sequence[int]) -> Tuple[int, int]:
        """Append pages whose packed rows were already written into ``tail``.  Returns (first id, count)."""
        lens = [int(x) for x in page_lens]
        need = int(nat.lib.b200ms_padded_rows(nat.i32_array(lens), len(lens)))
        if self._rows + need > self._cap_rows:
            raise ValueError("commit_rows: the rows were not written inside the block")
        first = self.n_pages
        self._rows += need
        self._page_lens.extend(lens)
        self._attached = False
        return first, len(lens)

    def add_pages(self, pages: Sequence[ArrayLike]) -> Tuple[int, int]:
        """Append pages ([P_i,128] float32/bfloat16; numpy on host or torch on either side).  Returns (first id, count).

        Mirrors the write half of store_embeddings (multi_vector_store.py:681-703 quantise+insert;
        fast_multivector_store.py:673-707 np.save of float32): one H2D copy of the ragged rows, one pack kernel.
        """
        if len(pages) == 0:
            return self.n_pages, 0
        lens = [int(p.shape[0]) for p in pages]
        for p in pages:
            if p.ndim != 2 or p.shape[1] != nat.DIM:
                raise ValueError(f"page embeddings must be [P,{nat.DIM}], got {tuple(p.shape)}")
        src, src_dtype = self._stage_rows(pages)
        lens_c = nat.i32_array(lens)
        nbytes = int(nat.lib.b200ms_padded_rows(lens_c, len(lens))) * self.row_bytes
        dst = self.tail(nbytes)
        # host tier: pack on the GPU into a device temporary, then one D2H copy into the block
        # (pages none of which has a row have no tail: the call then needs a destination all the same)
        packed = dst if dst.is_cuda and nbytes else torch.empty(max(nbytes, 1), dtype=torch.uint8, device=self.device)
        with torch.cuda.device(self.device):
            self.h.check(
                nat.lib.b200ms_pack_pages(self.h.ptr, _vp(src), src_dtype, lens_c, len(lens), _vp(packed), self.dtype,
                                          ctypes.c_float(self.i8_scale), self._stream()),
                "b200ms_pack_pages",
            )
        if packed is not dst:
            dst.copy_(packed[:nbytes])
        return self.commit_rows(lens)

    def _stage_rows(self, mats: Sequence[ArrayLike]) -> Tuple[torch.Tensor, int]:
        """Concatenate ragged [n_i,128] matrices into one device tensor (float32 or bfloat16)."""
        if all(isinstance(m, torch.Tensor) for m in mats):
            dt = torch.bfloat16 if all(m.dtype == torch.bfloat16 for m in mats) else torch.float32
            cat = torch.cat([m.to(device=self.device, dtype=dt) for m in mats], dim=0) if len(mats) > 1 else mats[0].to(
                device=self.device, dtype=dt)
            cat = cat.contiguous()
            if cat.shape[0] == 0:
                cat = torch.zeros((1, nat.DIM), dtype=dt, device=self.device)
            return cat, _check_queries(cat, (), self.device)
        mats = [np.asarray(m.cpu() if isinstance(m, torch.Tensor) else m, dtype=np.float32) for m in mats]
        total = int(sum(m.shape[0] for m in mats))
        if total == 0:
            return torch.zeros((1, nat.DIM), dtype=torch.float32, device=self.device), nat.F32
        if total < 256:  # queries, single small pages: a pageable copy is cheaper than touching the staging buffer
            return torch.from_numpy(np.ascontiguousarray(np.concatenate(mats, axis=0))).to(self.device), nat.F32
        # ingest: gather the ragged pages straight into a reusable PINNED staging buffer and copy once (pageable H2D
        # measured 2.6 GB/s through store_embeddings; the reference hands pages over as host float32, :673-707)
        pin = getattr(self, "_pin", None)
        if pin is None or pin.shape[0] < total:
            pin = self._pin = torch.empty((max(total, 1 << 15), nat.DIM), dtype=torch.float32).pin_memory()
        view = pin[:total].numpy()
        o = 0
        for m in mats:
            view[o:o + m.shape[0]] = m
            o += m.shape[0]
        dev = torch.empty((total, nat.DIM), dtype=torch.float32, device=self.device)
        dev.copy_(pin[:total], non_blocking=True)
        torch.cuda.current_stream(self.device).synchronize()  # the staging buffer is reused by the next call
        return dev, nat.F32

    def adopt_packed(self, rows: torch.Tensor, page_lens: Sequence[int]):
        """Use an already packed device buffer (uint8 view or typed tensor, 1024-byte aligned, layout as described in the
        class docstring) as the corpus without copying -- bench.py builds its synthetic shard this way."""
        if self.tier == "host":  # the rows move into a host block of exactly their size
            self.clear()
            self.reserve_rows(int(nat.lib.b200ms_padded_rows(nat.i32_array([int(x) for x in page_lens]), len(page_lens))))
            self.append_packed(rows, page_lens)
            return
        buf = rows.view(torch.uint8).reshape(-1)
        if buf.data_ptr() % 1024:
            raise ValueError("packed corpus must be 1024-byte aligned")
        lens = [int(x) for x in page_lens]
        lens_c = nat.i32_array(lens)
        need = int(nat.lib.b200ms_padded_rows(lens_c, len(lens)))
        if buf.numel() < need * self.row_bytes:
            raise ValueError("packed buffer smaller than the page lengths imply")
        if self._block is not None:  # the index's own block goes; work queued on its rows must be over first
            torch.cuda.synchronize(self.device)
            self._block.free()
            self._block = None
        self._buf, self._cap_rows, self._rows = buf, buf.numel() // self.row_bytes, need
        self._page_lens = lens
        self._attached = False

    def append_packed(self, rows: torch.Tensor, page_lens: Sequence[int]) -> Tuple[int, int]:
        """Append already packed rows (uint8 view of the corpus dtype's layout, pages padded to 32 rows) with one copy.
        Returns (first id, count)."""
        lens = [int(x) for x in page_lens]
        flat = rows.view(torch.uint8).reshape(-1)
        nbytes = int(nat.lib.b200ms_padded_rows(nat.i32_array(lens), len(lens))) * self.row_bytes
        if flat.numel() < nbytes:
            raise ValueError("packed buffer smaller than the page lengths imply")
        self.tail(nbytes).copy_(flat[:nbytes])
        return self.commit_rows(lens)

    def page_row_range(self, first: int, n: int) -> Tuple[int, int]:
        """Padded row range [r0, r1) that pages [first, first+n) occupy in the packed buffer."""
        pad = _padded_lens(self._page_lens)
        r0 = int(pad[:first].sum())
        return r0, r0 + int(pad[first:first + n].sum())

    def _attach(self):
        if self._attached:
            return
        lens_c = nat.i32_array(self._page_lens)
        with torch.cuda.device(self.device):
            torch.cuda.current_stream(self.device).synchronize()  # pack kernels ran on torch's stream
            if self.tier == "host":
                self.h.check(nat.lib.b200ms_set_corpus_host(self.h.ptr, _vp(self._buf) if self.n_pages else None, self.dtype,
                                                            lens_c, self.n_pages), "b200ms_set_corpus_host")
            else:
                self.h.check(nat.lib.b200ms_set_corpus(self.h.ptr, _vp(self._buf), self.dtype, lens_c, self.n_pages),
                             "b200ms_set_corpus")
        self._attached = True

    def clear(self):
        """Drop every page but keep the device buffer and the native handle (scratch indexes, e.g. the reranker's)."""
        self._rows = 0
        self._page_lens = []
        self._attached = False

    def compact(self, keep: Sequence[int]):
        """Keep only the pages in `keep` (ascending old ids), renumbering them 0..len(keep)-1, in place (DELETE ... WHERE
        document_id, multi_vector_store.py:929-933): the maximal runs of consecutive surviving pages move down inside the
        buffer -- on the GPU with one b200ms_compact_rows call, after which the block's freed tail goes back to the driver;
        on the host tier with one forward (overlap-safe) memmove per run."""
        keep = [int(p) for p in keep]
        lens = self._page_lens
        runs = _row_runs(lens, keep)
        new_rows = sum(b - a for a, b in runs)
        if self.tier == "host":
            self._host_barrier()
            base, dst = self._buf.data_ptr(), 0
            for a, b in runs:
                if dst != a * self.row_bytes:
                    ctypes.memmove(base + dst, base + a * self.row_bytes, (b - a) * self.row_bytes)
                dst += (b - a) * self.row_bytes
        elif self._buf is not None:
            if self._block is None:  # a caller's tensor (adopt_packed) is not compacted behind the caller's back
                self._resize_block(self._rows)
            _compact_rows(self.h, self.device, self._buf, self.row_bytes, runs)
            self._resize_block(new_rows)
        self._rows = new_rows
        self._page_lens = [lens[p] for p in keep]
        self._attached = False

    def packed_rows(self) -> torch.Tensor:
        """The packed corpus as a uint8 tensor [rows_padded, row_bytes] (a view; of host memory for the host tier)."""
        if self._buf is None:
            return torch.empty((0, self.row_bytes), dtype=torch.uint8, device=self.device if self.tier == "hbm" else "cpu")
        return self._buf[: self._rows * self.row_bytes].view(self._rows, self.row_bytes)

    def gather_stats(self) -> dict:
        """Of the last host-tier rerank call: unique pages gathered, bytes copied over PCIe (padded rows x row bytes),
        staging rounds, and the device time of the gather kernels (ms); synchronises."""
        u, b, r, ms = ctypes.c_int64(), ctypes.c_int64(), ctypes.c_int(), ctypes.c_float()
        self.h.check(nat.lib.b200ms_last_gather_stats(self.h.ptr, ctypes.byref(u), ctypes.byref(b), ctypes.byref(r),
                                                      ctypes.byref(ms)), "b200ms_last_gather_stats")
        return {"unique_pages": int(u.value), "bytes": int(b.value), "rounds": int(r.value), "ms": float(ms.value)}

    def scan_stats(self) -> dict:
        """Of the last full scan (score_groups or a search without candidates): work units and padded rows it walked -- the
        whole corpus, or only the pages its allow masks named; synchronises with that call."""
        u, r = ctypes.c_int64(), ctypes.c_int64()
        self.h.check(nat.lib.b200ms_last_scan_stats(self.h.ptr, ctypes.byref(u), ctypes.byref(r)), "b200ms_last_scan_stats")
        return {"units": int(u.value), "rows": int(r.value)}

    # ------------------------------------------------------------------ queries
    @staticmethod
    def _q_lens(queries: Sequence[ArrayLike]) -> List[int]:
        for q in queries:
            if q.ndim != 2 or q.shape[1] != nat.DIM:
                raise ValueError(f"query embeddings must be [T,{nat.DIM}], got {tuple(q.shape)}")
        return [int(q.shape[0]) for q in queries]

    def mask_from_pages(self, allowed: np.ndarray) -> np.ndarray:
        """bool[n_pages] -> uint32 bitmask words (bit p&31 of word p>>5), the device filter format."""
        allowed = np.asarray(allowed, dtype=bool)
        if allowed.shape[0] != self.n_pages:
            raise ValueError("mask length must equal n_pages")
        return PageCatalog.mask_words(allowed)

    def _check_mask(self, allow_mask) -> np.ndarray:
        return _host_mask_words(allow_mask, self.n_pages)

    def search_host(self, queries: Sequence[np.ndarray], k: int, allow_mask: Optional[np.ndarray] = None,
                    id_base: int = 0, out: Optional[Tuple[np.ndarray, np.ndarray, np.ndarray]] = None):
        """End-to-end query step from HOST buffers (float32 [T_i,128] each): H2D, pack, scan, top-k, D2H; synchronous.

        Returns (scores float32 [n_q,k], page ids int64 [n_q,k], counts int32 [n_q]); unused slots are -inf / -1.
        Replaces the scoring half of query_similar (multi_vector_store.py:721-763 / fast_multivector_store.py:553-557).
        """
        self._attach()
        lens = self._q_lens(queries)
        n_q = len(lens)
        if n_q == 1:
            q_host = np.ascontiguousarray(queries[0], dtype=np.float32)
        else:
            q_host = np.ascontiguousarray(np.concatenate([np.asarray(q, dtype=np.float32) for q in queries], axis=0))
        if out is None:
            out = (np.empty((n_q, k), np.float32), np.empty((n_q, k), np.int64), np.empty((n_q,), np.int32))
        ts, ti, tc = out
        mask_p = None
        if allow_mask is not None:
            allow_mask = self._check_mask(allow_mask)
            mask_p = allow_mask.ctypes.data_as(ctypes.c_void_p)
        self.h.check(
            nat.lib.b200ms_search_host(self.h.ptr, q_host.ctypes.data_as(ctypes.c_void_p), nat.i32_array(lens), n_q, int(k),
                                       mask_p, ctypes.c_float(self.i8_scale), ctypes.c_float(self.score_scale),
                                       int(id_base), ts.ctypes.data_as(ctypes.c_void_p),
                                       ti.ctypes.data_as(ctypes.c_void_p), tc.ctypes.data_as(ctypes.c_void_p)),
            "b200ms_search_host",
        )
        return ts, ti, tc

    def search_host_masked(self, queries: Sequence[np.ndarray], k: int, allow_masks: Sequence[Optional[np.ndarray]],
                           id_base: int = 0):
        """search_host with one allow-mask PER QUERY (``allow_masks[i]``: uint32 words as for ``allow_mask``, or None =
        unfiltered): queries of different users -- different authorised ``doc_ids`` (document_service.py:408-417) -- share one
        pass over the corpus.  Identical mask objects/contents are uploaded once."""
        self._attach()
        lens = self._q_lens(queries)
        n_q = len(lens)
        if len(allow_masks) != n_q:
            raise ValueError("one allow-mask (or None) per query")
        q_host = np.ascontiguousarray(np.concatenate([np.asarray(q, dtype=np.float32) for q in queries], axis=0))
        mat, index = PageCatalog.stack_masks([None if m is None else self._check_mask(m) for m in allow_masks])
        ts, ti, tc = np.empty((n_q, k), np.float32), np.empty((n_q, k), np.int64), np.empty((n_q,), np.int32)
        self.h.check(
            nat.lib.b200ms_search_host_masked(
                self.h.ptr, q_host.ctypes.data_as(ctypes.c_void_p), nat.i32_array(lens), n_q, int(k),
                None if mat is None else mat.ctypes.data_as(ctypes.c_void_p), 0 if mat is None else len(mat),
                nat.i32_array(index),
                ctypes.c_float(self.i8_scale), ctypes.c_float(self.score_scale), int(id_base),
                ts.ctypes.data_as(ctypes.c_void_p), ti.ctypes.data_as(ctypes.c_void_p), tc.ctypes.data_as(ctypes.c_void_p)),
            "b200ms_search_host_masked",
        )
        return ts, ti, tc

    def search_host_flat(self, q_host: Union[np.ndarray, torch.Tensor], q_lens: Sequence[int], k: int,
                         out_scores: torch.Tensor, out_ids: torch.Tensor, out_counts: torch.Tensor,
                         allow_mask: Optional[np.ndarray] = None, id_base: int = 0):
        """Same as search_host for callers that keep (pinned) host buffers: q_host is [sum T,128] float32.
        The ctypes argument objects of the previous call are reused when nothing changed (interactive callers repeat the
        same shapes; building them costs as much as the whole C call for a 100-page corpus)."""
        if not self._attached:
            self._attach()
        qp = q_host.data_ptr() if isinstance(q_host, torch.Tensor) else q_host.ctypes.data
        mask_p = None
        if allow_mask is not None:
            allow_mask = self._check_mask(allow_mask)
            mask_p = allow_mask.ctypes.data_as(ctypes.c_void_p)
        key = (tuple(q_lens), int(k), int(id_base), out_scores.data_ptr(), out_ids.data_ptr(), out_counts.data_ptr())
        cached = getattr(self, "_flat_args", None)
        if cached is None or cached[0] != key:
            cached = (key, nat.i32_array(q_lens), ctypes.c_float(self.i8_scale), ctypes.c_float(self.score_scale),
                      ctypes.c_void_p(out_scores.data_ptr()), ctypes.c_void_p(out_ids.data_ptr()),
                      ctypes.c_void_p(out_counts.data_ptr()))
            self._flat_args = cached
        _, lens_c, c_scale, c_sscale, p_s, p_i, p_c = cached
        rc = nat.lib.b200ms_search_host(self.h.ptr, qp, lens_c, len(q_lens), key[1], mask_p, c_scale, c_sscale, key[2], p_s, p_i, p_c)
        if rc != 0:
            self.h.check(rc, "b200ms_search_host")

    def search_device(self, q_dev: torch.Tensor, q_lens: Sequence[int], k: int, allow_mask_dev: Optional[torch.Tensor] = None,
                      id_base: int = 0, out: Optional[Tuple[torch.Tensor, torch.Tensor, torch.Tensor]] = None,
                      mask_index_dev: Optional[torch.Tensor] = None):
        """Asynchronous search with device-resident queries ([sum T,128] float32|bfloat16) on torch's current stream.

        ``allow_mask_dev``: one mask (int32/uint32 words) for every query, or -- with ``mask_index_dev`` (int32 [n_q], -1 =
        unfiltered) -- a [n_masks, words] matrix with one row per distinct filter (b200ms_search_device_masked)."""
        n_q = len(q_lens)
        q_dtype = _check_queries(q_dev, q_lens, self.device)
        masks, n_masks, index = _check_device_masks(allow_mask_dev, mask_index_dev, n_q, self.n_pages, self.device)
        ts, ti, tc = _topk_outputs(n_q, int(k), self.device, out)
        self._attach()
        if index is not None:
            with torch.cuda.device(self.device):
                self.h.check(
                    nat.lib.b200ms_search_device_masked(
                        self.h.ptr, _vp(q_dev), q_dtype, nat.i32_array(q_lens), n_q, int(k), _vp(masks), n_masks, _vp(index),
                        ctypes.c_float(self.i8_scale), ctypes.c_float(self.score_scale), int(id_base), _vp(ts), _vp(ti),
                        _vp(tc), self._stream()),
                    "b200ms_search_device_masked",
                )
            return ts, ti, tc
        with torch.cuda.device(self.device):
            self.h.check(
                nat.lib.b200ms_search_device(self.h.ptr, _vp(q_dev), q_dtype, nat.i32_array(q_lens), n_q, int(k), _vp(masks),
                                             ctypes.c_float(self.i8_scale), ctypes.c_float(self.score_scale), int(id_base),
                                             _vp(ts), _vp(ti), _vp(tc), self._stream()),
                "b200ms_search_device",
            )
        return ts, ti, tc

    def score_groups(self, queries: Sequence[ArrayLike]):
        """Raw kernel output for tests and diagnostics: (group_scores tensor [n_groups_padded, ld] float32|int32,
        group_offsets int32 [n_q+1], n_pages).  Calls pack_queries + score through the C-ABI."""
        self._attach()
        lens = self._q_lens(queries)
        n_q = len(lens)
        src, src_dtype = self._stage_rows(queries)
        lens_c = nat.i32_array(lens)
        groups = int(nat.lib.b200ms_query_groups(lens_c, n_q))
        gp = max((groups + 3) // 4 * 4, 4)
        q_packed = _aligned_bytes(gp * 32 * self.row_bytes, self.device)
        goff = (ctypes.c_int32 * (n_q + 1))()
        ng = ctypes.c_int(0)
        ld = (self.n_pages + 31) // 32 * 32
        sdt = torch.float32 if self.float_scores else torch.int32
        scores = torch.zeros((gp, max(ld, 32)), dtype=sdt, device=self.device)
        with torch.cuda.device(self.device):
            self.h.check(
                nat.lib.b200ms_pack_queries(self.h.ptr, _vp(src), src_dtype, lens_c, n_q, _vp(q_packed), self.dtype,
                                            ctypes.c_float(self.i8_scale), goff, ctypes.byref(ng), self._stream()),
                "b200ms_pack_queries",
            )
            self.h.check(
                nat.lib.b200ms_score(self.h.ptr, _vp(q_packed), ng.value, lens_c, goff, n_q, _vp(scores), max(ld, 32),
                                     self._stream()),
                "b200ms_score",
            )
        return scores, np.asarray(list(goff), dtype=np.int32), self.n_pages, q_packed

    def score_matrix(self, queries: Sequence[ArrayLike]) -> np.ndarray:
        """[n_q, n_pages] scores on the reference's scale (float64 on host; the per-query sum over 32-token groups is done
        here in float64 for diagnostics only -- the product path sums inside the top-k kernel)."""
        scores, goff, n_pages, _ = self.score_groups(queries)
        torch.cuda.synchronize(self.device)
        s = scores[:, :n_pages].cpu().numpy().astype(np.float64)
        out = np.zeros((len(goff) - 1, n_pages), dtype=np.float64)
        for q in range(len(goff) - 1):
            out[q] = s[goff[q]:goff[q + 1]].sum(axis=0) * self.score_scale
        return out

    def sign_pack(self, x: ArrayLike) -> torch.Tensor:
        """[n,128] float32/bfloat16 -> uint8 [n,16] MSB-first sign bits on the device (fast_ops.binary_quantize_packed)."""
        src, src_dtype = self._stage_rows([x])
        n = int(x.shape[0])
        out = torch.empty((max(n, 1), 16), dtype=torch.uint8, device=self.device)
        with torch.cuda.device(self.device):
            self.h.check(nat.lib.b200ms_sign_pack(self.h.ptr, _vp(src), src_dtype, n, _vp(out), self._stream()),
                         "b200ms_sign_pack")
        return out[:n]

    def hamming_distance_batch(self, query_bits, candidate_bits) -> torch.Tensor:
        """fast_ops.hamming_distance_batch on the device: packed 16-byte query (bytes / uint8[16]) vs packed candidates
        (list of bytes / uint8 [n,16]) -> int32 tensor [n] of Hamming distances."""
        q = np.frombuffer(bytes(query_bits), dtype=np.uint8) if isinstance(query_bits, (bytes, bytearray)) else np.asarray(query_bits, np.uint8)
        if isinstance(candidate_bits, (list, tuple)):
            lens = {len(c) for c in candidate_bits}
            if lens - {16}:
                raise ValueError(f"Vector length mismatch: candidates must be 16 bytes like the query, got {sorted(lens)}")
            c = np.frombuffer(b"".join(bytes(x) for x in candidate_bits), dtype=np.uint8).reshape(-1, 16)
        else:
            c = candidate_bits
        if q.size != 16:
            raise ValueError(f"Vector length mismatch: {q.size} vs 16")  # ValueError like the Rust implementation
        qd = torch.from_numpy(q.reshape(16).copy()).to(self.device)
        cd = c if isinstance(c, torch.Tensor) else torch.from_numpy(np.ascontiguousarray(c, dtype=np.uint8)).to(self.device)
        cd = cd.contiguous().view(-1, 16)
        qa = _aligned_bytes(16, self.device, 16); qa.copy_(qd)
        ca = _aligned_bytes(max(cd.numel(), 16), self.device, 16); ca[: cd.numel()].copy_(cd.reshape(-1))
        out = torch.empty((cd.shape[0],), dtype=torch.int32, device=self.device)
        with torch.cuda.device(self.device):
            self.h.check(nat.lib.b200ms_hamming_batch(self.h.ptr, _vp(qa), _vp(ca), cd.shape[0], _vp(out), self._stream()),
                         "b200ms_hamming_batch")
        return out

    def merge_topk(self, cand_scores: torch.Tensor, cand_ids: torch.Tensor, k: int):
        """Merge candidate lists [n_q, m] (ids < 0 ignored) -> top-k by (score desc, id asc), on the device."""
        n_q, m = cand_scores.shape
        ts, ti, tc = _topk_outputs(n_q, int(k), self.device)
        with torch.cuda.device(self.device):
            self.h.check(
                nat.lib.b200ms_merge_topk(self.h.ptr, _vp(cand_scores.contiguous()), _vp(cand_ids.contiguous()), n_q, m, int(k),
                                          _vp(ts), _vp(ti), _vp(tc), self._stream()),
                "b200ms_merge_topk",
            )
        return ts, ti, tc

    # ------------------------------------------------------------------ candidate rerank (two-stage search)
    def rerank(self, q_dev: torch.Tensor, q_lens: Sequence[int], cand_ids: torch.Tensor, k: int):
        """Exact MaxSim of every query over ONE shared candidate list: cand_ids int64 [n_cand] on the device (-1 = unused
        slot) -> (scores [n_q,k], page ids [n_q,k], counts [n_q]) on the device (b200ms_rerank_device)."""
        n_q = len(q_lens)
        q_dtype = _check_queries(q_dev, q_lens, self.device)
        n_cand, kk = _check_candidates(cand_ids, n_q, k, self.device, per_query=False)
        ts, ti, tc = _topk_outputs(n_q, kk, self.device)
        self._attach()
        with torch.cuda.device(self.device):
            self.h.check(
                nat.lib.b200ms_rerank_device(self.h.ptr, _vp(q_dev), q_dtype, nat.i32_array(q_lens), n_q, _vp(cand_ids), n_cand, kk,
                                             ctypes.c_float(self.i8_scale), ctypes.c_float(self.score_scale), _vp(ts), _vp(ti),
                                             _vp(tc), self._stream()),
                "b200ms_rerank_device")
        return ts, ti, tc

    def rerank_batch(self, q_dev: torch.Tensor, q_lens: Sequence[int], cand_ids: torch.Tensor, k: int,
                     out: Optional[Tuple[torch.Tensor, torch.Tensor, torch.Tensor]] = None):
        """Exact MaxSim of every query over ITS OWN candidate list: cand_ids int64 [n_q, n_cand] on the device (-1 = unused
        slot) -> (scores [n_q,k], page ids [n_q,k], counts [n_q]) on the device; one call for the whole batch
        (b200ms_rerank_batch_device; fast_multivector_store.py:545-557 does this one query at a time on <= 75 pages)."""
        n_q = len(q_lens)
        q_dtype = _check_queries(q_dev, q_lens, self.device)
        n_cand, kk = _check_candidates(cand_ids, n_q, k, self.device, per_query=True)
        ts, ti, tc = _topk_outputs(n_q, kk, self.device, out)
        self._attach()
        with torch.cuda.device(self.device):
            self.h.check(
                nat.lib.b200ms_rerank_batch_device(self.h.ptr, _vp(q_dev), q_dtype, nat.i32_array(q_lens), n_q, _vp(cand_ids),
                                                   n_cand, kk,
                                                   ctypes.c_float(self.i8_scale), ctypes.c_float(self.score_scale), _vp(ts),
                                                   _vp(ti), _vp(tc), self._stream()),
                "b200ms_rerank_batch_device")
        return ts, ti, tc

    # ------------------------------------------------------------------ stored pages as the queries
    def _src_pages(self, src_pages) -> List[int]:
        """Source page ids -> a non-empty list of ints in [0, n_pages) (ValueError otherwise, before any launch)."""
        ids = [int(p) for p in (src_pages.tolist() if isinstance(src_pages, (np.ndarray, torch.Tensor)) else src_pages)]
        if not ids or any(not 0 <= p < self.n_pages for p in ids):
            raise ValueError(f"src_pages must be one or more page ids in [0, {self.n_pages}), got {ids}")
        return ids

    def search_pages(self, src_pages, k: int, allow_mask_dev: Optional[torch.Tensor] = None,
                     mask_index_dev: Optional[torch.Tensor] = None, id_base: int = 0,
                     out: Optional[Tuple[torch.Tensor, torch.Tensor, torch.Tensor]] = None):
        """Pages like stored pages (b200ms_search_pages_device), asynchronous on torch's current stream: source page i's own
        packed rows are query i of a full scan, and a page's score is the page-to-page MaxSim per source row -- the score
        search_device would give the source's rows, over the source's row count.  Masks as search_device, one row per source
        (the only filter: the source itself is returned unless its mask bit is clear).  A source without rows gets count 0.
        Returns device tensors (scores float32 [n_src,k], page ids + id_base int64 [n_src,k], counts int32 [n_src])."""
        ids = self._src_pages(src_pages)
        masks, n_masks, index = _check_device_masks(allow_mask_dev, mask_index_dev, len(ids), self.n_pages, self.device)
        if masks is not None and index is None:  # one mask for every source: a one-row matrix
            index = torch.zeros((len(ids),), dtype=torch.int32, device=self.device)
        ts, ti, tc = _topk_outputs(len(ids), int(k), self.device, out)
        self._attach()
        with torch.cuda.device(self.device):
            self.h.check(
                nat.lib.b200ms_search_pages_device(
                    self.h.ptr, nat.i64_array(ids), len(ids), int(k), _vp(masks), n_masks, _vp(index),
                    ctypes.c_float(self.score_scale), int(id_base), _vp(ts), _vp(ti), _vp(tc), self._stream()),
                "b200ms_search_pages_device")
        return ts, ti, tc

    def rerank_pages_batch(self, src_pages, cand_ids: torch.Tensor, k: int, allow_mask_dev: Optional[torch.Tensor] = None,
                           mask_index_dev: Optional[torch.Tensor] = None,
                           out: Optional[Tuple[torch.Tensor, torch.Tensor, torch.Tensor]] = None):
        """rerank_batch with stored pages as the queries (b200ms_rerank_pages_batch_device): source i's packed rows against
        its own candidate list cand_ids int64 [n_src, n_cand] (-1 = unused slot), scores as search_pages; a candidate its
        source's mask row forbids is an unused slot.  k is capped at n_cand.  Works on both tiers."""
        ids = self._src_pages(src_pages)
        n_cand, kk = _check_candidates(cand_ids, len(ids), k, self.device, per_query=True)
        masks, n_masks, index = _check_device_masks(allow_mask_dev, mask_index_dev, len(ids), self.n_pages, self.device)
        if masks is not None and index is None:
            index = torch.zeros((len(ids),), dtype=torch.int32, device=self.device)
        ts, ti, tc = _topk_outputs(len(ids), kk, self.device, out)
        self._attach()
        with torch.cuda.device(self.device):
            self.h.check(
                nat.lib.b200ms_rerank_pages_batch_device(
                    self.h.ptr, nat.i64_array(ids), len(ids), _vp(cand_ids), n_cand, kk, _vp(masks), n_masks, _vp(index),
                    ctypes.c_float(self.score_scale), _vp(ts), _vp(ti), _vp(tc), self._stream()),
                "b200ms_rerank_pages_batch_device")
        return ts, ti, tc

    def page_rows(self, src_pages) -> Tuple[torch.Tensor, List[int]]:
        """The true rows of the source pages back to back as float32 [sum len, 128] on the device, dequantised
        (b200ms_page_rows_device: int8 codes and e4m3 values over the corpus scale, sign bits as +-1), and their lengths --
        the float query of a first stage."""
        ids = self._src_pages(src_pages)
        lens = [int(self._page_lens[p]) for p in ids]
        out = torch.empty((max(sum(lens), 1), nat.DIM), dtype=torch.float32, device=self.device)
        scale = 1.0 / self.i8_scale if self.dtype in (nat.I8, nat.F8) else 1.0
        self._attach()
        with torch.cuda.device(self.device):
            self.h.check(nat.lib.b200ms_page_rows_device(self.h.ptr, nat.i64_array(ids), len(ids), ctypes.c_float(scale),
                                                         _vp(out), self._stream()), "b200ms_page_rows_device")
        return out, lens

    # ------------------------------------------------------------------ relevance feedback: weighted examples
    def _examples(self, q_dev: Optional[torch.Tensor], q_lens: Sequence[int], ex_pages, ex_req: Sequence[int],
                  ex_weights: Sequence[float], n_req: int):
        """Checked examples of a request batch (ValueError before any launch): n_qe query embeddings (rows of q_dev, lengths
        q_lens), then stored pages ex_pages; example i belongs to request ex_req[i] and weighs ex_weights[i] (finite and
        non-zero in float32), and every request has an example of positive weight.  Returns (q dtype code, q_lens, page
        ids, ex_req, float32 weights)."""
        q_lens = [int(n) for n in q_lens]
        pages = [int(p) for p in (ex_pages.tolist() if isinstance(ex_pages, (np.ndarray, torch.Tensor)) else ex_pages)]
        req = [int(r) for r in ex_req]
        w = np.asarray(list(ex_weights), dtype=np.float32)
        n_ex, n_req = len(q_lens) + len(pages), int(n_req)
        if n_ex < 1 or n_req < 1 or len(req) != n_ex or w.shape != (n_ex,):
            raise ValueError(f"examples: {len(q_lens)} query + {len(pages)} page examples need one request and one weight "
                             f"each (got {len(req)} and {w.size}), n_req >= 1")
        if any(n < 0 for n in q_lens):
            raise ValueError(f"q_lens must be >= 0, got {q_lens}")
        if q_lens and q_dev is None:
            raise ValueError("query examples need their rows: q_dev is None")
        q_dtype = _check_queries(q_dev, q_lens, self.device) if q_lens else nat.F32
        if any(not 0 <= p < self.n_pages for p in pages):
            raise ValueError(f"example pages must be page ids in [0, {self.n_pages}), got {pages}")
        if any(not 0 <= r < n_req for r in req):
            raise ValueError(f"ex_req must name requests in [0, {n_req}), got {req}")
        if not np.all(np.isfinite(w)) or np.any(w == 0):
            raise ValueError(f"example weights must be finite and non-zero in float32, got {w.tolist()}")
        if len({r for r, x in zip(req, w) if x > 0}) != n_req:
            raise ValueError("every request needs an example of positive weight")
        return q_dtype, q_lens, pages, req, w

    def _request_masks(self, allow_mask_dev, mask_index_dev, n_req: int):
        masks, n_masks, index = _check_device_masks(allow_mask_dev, mask_index_dev, n_req, self.n_pages, self.device)
        if masks is not None and index is None:  # one mask for every request: a one-row matrix
            index = torch.zeros((n_req,), dtype=torch.int32, device=self.device)
        return masks, n_masks, index

    def search_examples(self, q_dev: Optional[torch.Tensor], q_lens: Sequence[int], ex_pages, ex_req: Sequence[int],
                        ex_weights: Sequence[float], n_req: int, k: int, allow_mask_dev: Optional[torch.Tensor] = None,
                        mask_index_dev: Optional[torch.Tensor] = None, id_base: int = 0,
                        out: Optional[Tuple[torch.Tensor, torch.Tensor, torch.Tensor]] = None):
        """Relevance feedback (b200ms_search_examples_device), asynchronous on torch's current stream: each of n_req requests
        ranks pages by the weighted sum of their scores against its examples, all examples scored in one full scan.
        Examples: query embeddings (q_dev [sum q_lens, 128] float32 | bfloat16, or None without query examples), then stored
        page ids ``ex_pages``; ``ex_req`` / ``ex_weights`` give each one's request and weight (> 0 like, < 0 unlike).  An
        example's score is the page-to-page scale of search_pages: the MaxSim per example row (or token).  Masks as
        search_device, one row per REQUEST; example pages are returned unless their bits are clear.  Returns device tensors
        (scores float32 [n_req,k], page ids + id_base int64 [n_req,k], counts int32 [n_req])."""
        q_dtype, q_lens, pages, req, w = self._examples(q_dev, q_lens, ex_pages, ex_req, ex_weights, n_req)
        masks, n_masks, index = self._request_masks(allow_mask_dev, mask_index_dev, int(n_req))
        ts, ti, tc = _topk_outputs(int(n_req), int(k), self.device, out)
        self._attach()
        with torch.cuda.device(self.device):
            self.h.check(
                nat.lib.b200ms_search_examples_device(
                    self.h.ptr, _vp(q_dev) if q_lens else None, q_dtype, nat.i32_array(q_lens), len(q_lens),
                    nat.i64_array(pages), len(pages), nat.i32_array(req), nat.f32_array(w), int(n_req), int(k), _vp(masks),
                    n_masks, _vp(index), ctypes.c_float(self.i8_scale), ctypes.c_float(self.score_scale), int(id_base),
                    _vp(ts), _vp(ti), _vp(tc), self._stream()),
                "b200ms_search_examples_device")
        return ts, ti, tc

    def rerank_examples_batch(self, q_dev: Optional[torch.Tensor], q_lens: Sequence[int], ex_pages, ex_req: Sequence[int],
                              ex_weights: Sequence[float], n_req: int, cand_ids: torch.Tensor, k: int,
                              allow_mask_dev: Optional[torch.Tensor] = None, mask_index_dev: Optional[torch.Tensor] = None,
                              out: Optional[Tuple[torch.Tensor, torch.Tensor, torch.Tensor]] = None):
        """search_examples over one candidate list per request, cand_ids int64 [n_req, n_cand] (-1 = unused slot;
        b200ms_rerank_examples_batch_device): every example of request r scores r's list, ties go to the lower slot, and a
        candidate r's mask row forbids is an unused slot.  k is capped at n_cand.  Works on both tiers."""
        q_dtype, q_lens, pages, req, w = self._examples(q_dev, q_lens, ex_pages, ex_req, ex_weights, n_req)
        n_cand, kk = _check_candidates(cand_ids, int(n_req), k, self.device, per_query=True)
        masks, n_masks, index = self._request_masks(allow_mask_dev, mask_index_dev, int(n_req))
        ts, ti, tc = _topk_outputs(int(n_req), kk, self.device, out)
        self._attach()
        with torch.cuda.device(self.device):
            self.h.check(
                nat.lib.b200ms_rerank_examples_batch_device(
                    self.h.ptr, _vp(q_dev) if q_lens else None, q_dtype, nat.i32_array(q_lens), len(q_lens),
                    nat.i64_array(pages), len(pages), nat.i32_array(req), nat.f32_array(w), int(n_req), _vp(cand_ids),
                    n_cand, kk, _vp(masks), n_masks, _vp(index), ctypes.c_float(self.i8_scale),
                    ctypes.c_float(self.score_scale), _vp(ts), _vp(ti), _vp(tc), self._stream()),
                "b200ms_rerank_examples_batch_device")
        return ts, ti, tc

    def union_candidates(self, cand_ids: torch.Tensor, list_off: Sequence[int], width: Optional[int] = None) -> torch.Tensor:
        """Union of first-stage lists on the device (b200ms_union_candidates_device), asynchronous: request r owns rows
        list_off[r] .. list_off[r+1] of cand_ids int64 [n_lists, n_cand]; returns int64 [n_req, width] with r's distinct page
        ids (negative ids are unused slots) in first-occurrence order, row-major over its lists, -1 padded.  ``width``
        defaults to the most slots any request owns (nothing is cut)."""
        off = [int(o) for o in list_off]
        n_lists = int(cand_ids.shape[0]) if cand_ids.ndim == 2 else -1
        if (cand_ids.dtype != torch.int64 or cand_ids.ndim != 2 or not cand_ids.is_contiguous() or cand_ids.device != self.device
                or cand_ids.shape[1] < 1):
            raise ValueError(f"cand_ids must be a contiguous int64 [n_lists, n_cand >= 1] tensor on {self.device}")
        if len(off) < 2 or off[0] != 0 or off[-1] != n_lists or any(b < a for a, b in zip(off, off[1:])):
            raise ValueError(f"list_off must rise from 0 to n_lists = {n_lists}, got {off}")
        n_cand = int(cand_ids.shape[1])
        width = int(width) if width is not None else max(1, max(b - a for a, b in zip(off, off[1:])) * n_cand)
        if width < 1:
            raise ValueError(f"width must be >= 1, got {width}")
        out = torch.empty((len(off) - 1, width), dtype=torch.int64, device=self.device)
        with torch.cuda.device(self.device):
            self.h.check(
                nat.lib.b200ms_union_candidates_device(self.h.ptr, _vp(cand_ids), n_lists, n_cand, nat.i32_array(off),
                                                       len(off) - 1, _vp(out), width, self._stream()),
                "b200ms_union_candidates_device")
        return out

    # ------------------------------------------------------------------ grouping results by document
    def _check_docs_args(self, per_doc: int, page_doc_dev: torch.Tensor):
        if not 1 <= int(per_doc) <= nat.MAX_PER_DOC:
            raise ValueError(f"per_doc must be in [1, {nat.MAX_PER_DOC}]")
        if (page_doc_dev.dtype != torch.int32 or page_doc_dev.shape != (self.n_pages,) or not page_doc_dev.is_contiguous()
                or page_doc_dev.device != self.device):
            raise ValueError(f"page_doc_dev must be a contiguous int32 [{self.n_pages}] tensor on {self.device}")

    def search_docs_device(self, q_dev: torch.Tensor, q_lens: Sequence[int], k: int, per_doc: int, page_doc_dev: torch.Tensor,
                           n_docs: int, allow_mask_dev: Optional[torch.Tensor] = None,
                           mask_index_dev: Optional[torch.Tensor] = None, id_base: int = 0):
        """The top k DOCUMENTS instead of the top k pages (b200ms_search_docs_device), asynchronous on torch's current stream.

        page_doc_dev: int32 [n_pages] document ordinal of every page (a value outside [0, n_docs) hides the page).  Documents
        come in the order of their best page in search_device's ranking, each with its best ``per_doc`` pages in that
        ranking and their search_device scores.  Masks as search_device.  Returns device tensors (scores float32
        [n_q,k,per_doc], page ids + id_base int64 [n_q,k,per_doc], pages per document int32 [n_q,k], documents int32 [n_q]);
        unused entries are -inf / -1 / 0."""
        n_q = len(q_lens)
        q_dtype = _check_queries(q_dev, q_lens, self.device)
        self._check_docs_args(per_doc, page_doc_dev)
        masks, n_masks, index = _check_device_masks(allow_mask_dev, mask_index_dev, n_q, self.n_pages, self.device)
        ts, ti, pc, dc = _topk_outputs(n_q, int(k), self.device, per_doc=int(per_doc))
        if masks is not None and index is None:  # one mask for every query: a one-row matrix
            index = torch.zeros((n_q,), dtype=torch.int32, device=self.device)
        self._attach()
        with torch.cuda.device(self.device):
            self.h.check(
                nat.lib.b200ms_search_docs_device(
                    self.h.ptr, _vp(q_dev), q_dtype, nat.i32_array(q_lens), n_q, int(k), int(per_doc), _vp(page_doc_dev),
                    int(n_docs), _vp(masks), n_masks, _vp(index), ctypes.c_float(self.i8_scale),
                    ctypes.c_float(self.score_scale), int(id_base), _vp(ts), _vp(ti), _vp(pc), _vp(dc), self._stream()),
                "b200ms_search_docs_device")
        return ts, ti, pc, dc

    def search_docs(self, queries: Sequence[ArrayLike], k: int, per_doc: int, page_doc_dev: torch.Tensor, n_docs: int,
                    allow_mask: Optional[np.ndarray] = None):
        """search_docs_device from host query matrices and an optional host allow mask (uint32 words); synchronous, returns
        host arrays."""
        lens = self._q_lens(queries)
        src, _ = self._stage_rows(list(queries))
        mask_dev = _host_mask_to_device(allow_mask, self.n_pages, self.device)
        out = self.search_docs_device(src, lens, k, per_doc, page_doc_dev, n_docs, allow_mask_dev=mask_dev)
        return tuple(t.cpu().numpy() for t in out)

    def rerank_docs_batch(self, q_dev: torch.Tensor, q_lens: Sequence[int], cand_ids: torch.Tensor, k: int, per_doc: int,
                          page_doc_dev: torch.Tensor, n_docs: int):
        """rerank_batch grouped by document (b200ms_rerank_docs_batch_device): each query's own candidate list cand_ids int64
        [n_q, n_cand] (-1 = unused slot) is ranked as rerank_batch ranks it, and a page listed in several slots counts once,
        at its earliest slot.  k is capped at n_cand.  Outputs as search_docs_device."""
        n_q = len(q_lens)
        q_dtype = _check_queries(q_dev, q_lens, self.device)
        n_cand, kk = _check_candidates(cand_ids, n_q, k, self.device, per_query=True)
        self._check_docs_args(per_doc, page_doc_dev)
        ts, ti, pc, dc = _topk_outputs(n_q, kk, self.device, per_doc=int(per_doc))
        self._attach()
        with torch.cuda.device(self.device):
            self.h.check(
                nat.lib.b200ms_rerank_docs_batch_device(
                    self.h.ptr, _vp(q_dev), q_dtype, nat.i32_array(q_lens), n_q, _vp(cand_ids), n_cand, kk, int(per_doc),
                    _vp(page_doc_dev), int(n_docs), ctypes.c_float(self.i8_scale), ctypes.c_float(self.score_scale), _vp(ts),
                    _vp(ti), _vp(pc), _vp(dc), self._stream()),
                "b200ms_rerank_docs_batch_device")
        return ts, ti, pc, dc

    # ------------------------------------------------------------------ documents as one bag of patches
    def _doc_maxsim_args(self, q_dev, q_lens, k, per_doc, page_doc_dev, allow_mask_dev, mask_index_dev):
        if self.tier == "host":
            raise ValueError("document-level MaxSim reads every page of a document: it needs an HBM-tier index")
        n_q = len(q_lens)
        q_dtype = _check_queries(q_dev, q_lens, self.device)
        self._check_docs_args(per_doc, page_doc_dev)
        masks, n_masks, index = _check_device_masks(allow_mask_dev, mask_index_dev, n_q, self.n_pages, self.device)
        if masks is not None and index is None:  # one mask for every query: a one-row matrix
            index = torch.zeros((n_q,), dtype=torch.int32, device=self.device)
        ds, di, dc = _topk_outputs(n_q, int(k), self.device)
        es, ei, ec, _ = _topk_outputs(n_q, int(k), self.device, per_doc=int(per_doc))
        return q_dtype, masks, n_masks, index, (ds, di, ei, es, ec, dc)

    def search_doc_maxsim_device(self, q_dev: torch.Tensor, q_lens: Sequence[int], k: int, per_doc: int,
                                 page_doc_dev: torch.Tensor, n_docs: int, allow_mask_dev: Optional[torch.Tensor] = None,
                                 mask_index_dev: Optional[torch.Tensor] = None, id_base: int = 0):
        """The top k documents by document-level MaxSim (b200ms_search_doc_maxsim_device), asynchronous on torch's current
        stream: a document scores sum over the query's tokens of each token's best patch on ANY of its pages, so a query
        answered by several pages of one document ranks that document as one match.  Long documents are favoured (the
        score only grows with pages); nothing normalises it.

        page_doc_dev / masks as search_docs_device.  Returns device tensors: document scores float32 [n_q,k], document
        ordinals int64 [n_q,k], evidence page ids + id_base int64 [n_q,k,per_doc], evidence shares float32 [n_q,k,per_doc]
        (the token maxima each page holds; largest first), evidence pages int32 [n_q,k], documents found int32 [n_q];
        unused entries are -inf / -1 / 0.  An HBM-tier index only (ValueError on the host tier)."""
        q_dtype, masks, n_masks, index, out = self._doc_maxsim_args(q_dev, q_lens, k, per_doc, page_doc_dev, allow_mask_dev,
                                                                    mask_index_dev)
        self._attach()
        with torch.cuda.device(self.device):
            self.h.check(
                nat.lib.b200ms_search_doc_maxsim_device(
                    self.h.ptr, _vp(q_dev), q_dtype, nat.i32_array(q_lens), len(q_lens), int(k), int(per_doc),
                    _vp(page_doc_dev), int(n_docs), _vp(masks), n_masks, _vp(index), ctypes.c_float(self.i8_scale),
                    ctypes.c_float(self.score_scale), int(id_base), *[_vp(t) for t in out], self._stream()),
                "b200ms_search_doc_maxsim_device")
        ds, di, ei, es, ec, dc = out
        return ds, di, ei, es, ec, dc

    def search_doc_maxsim(self, queries: Sequence[ArrayLike], k: int, per_doc: int, page_doc_dev: torch.Tensor, n_docs: int,
                          allow_mask: Optional[np.ndarray] = None):
        """search_doc_maxsim_device from host query matrices and an optional host allow mask (uint32 words); synchronous,
        returns host arrays."""
        lens = self._q_lens(queries)
        src, _ = self._stage_rows(list(queries))
        mask_dev = _host_mask_to_device(allow_mask, self.n_pages, self.device)
        out = self.search_doc_maxsim_device(src, lens, k, per_doc, page_doc_dev, n_docs, allow_mask_dev=mask_dev)
        return tuple(t.cpu().numpy() for t in out)

    def rerank_doc_maxsim_batch(self, q_dev: torch.Tensor, q_lens: Sequence[int], cand_ids: torch.Tensor, k: int,
                                per_doc: int, page_doc_dev: torch.Tensor, n_docs: int,
                                allow_mask_dev: Optional[torch.Tensor] = None, mask_index_dev: Optional[torch.Tensor] = None,
                                id_base: int = 0):
        """search_doc_maxsim_device over the documents of each query's own first-stage pages, cand_ids int64 [n_q, n_cand]
        (-1 = unused slot; b200ms_rerank_doc_maxsim_batch_device): every allowed page of those documents is scored, not only
        the candidates.  Outputs as search_doc_maxsim_device."""
        _check_candidates(cand_ids, len(q_lens), k, self.device, per_query=True)
        q_dtype, masks, n_masks, index, out = self._doc_maxsim_args(q_dev, q_lens, k, per_doc, page_doc_dev, allow_mask_dev,
                                                                    mask_index_dev)
        self._attach()
        with torch.cuda.device(self.device):
            self.h.check(
                nat.lib.b200ms_rerank_doc_maxsim_batch_device(
                    self.h.ptr, _vp(q_dev), q_dtype, nat.i32_array(q_lens), len(q_lens), _vp(cand_ids),
                    int(cand_ids.shape[1]), int(k), int(per_doc), _vp(page_doc_dev), int(n_docs), _vp(masks), n_masks,
                    _vp(index), ctypes.c_float(self.i8_scale), ctypes.c_float(self.score_scale), int(id_base),
                    *[_vp(t) for t in out], self._stream()),
                "b200ms_rerank_doc_maxsim_batch_device")
        ds, di, ei, es, ec, dc = out
        return ds, di, ei, es, ec, dc

    # ------------------------------------------------------------------ explaining a match
    def explain(self, queries: Sequence[ArrayLike], page_ids, map_rows: int = 0):
        """Why pages matched: per query token, the best patch row of each named page and its similarity, computed with the
        search's own arithmetic on the packed rows (b200ms_explain_device), so the token scores add up to the page's score.

        queries: [T_i,128] float32/bfloat16 matrices (numpy or torch, either side).  page_ids: int64 [n_q, n_cand] (one list
        per query) or [n_cand] (shared by every query); -1 or an id outside [0, n_pages) is an unused slot.
        Returns device tensors (token_scores float32 [n_q, n_cand, T_max], best_rows int32 [n_q, n_cand, T_max],
        sim_map float32 [n_q, n_cand, T_max, map_rows] or None when map_rows == 0), in the units of the reported scores.
        best_rows index the page's rows in the order they were added; unused slots, empty pages and tokens past a query's
        length hold 0 / -1 / -inf, as do map rows past a page's length.  Works on both tiers."""
        self._attach()
        lens = self._q_lens(queries)
        n_q = len(lens)
        ids = page_ids if isinstance(page_ids, torch.Tensor) else torch.from_numpy(np.asarray(page_ids, dtype=np.int64))
        ids = ids.to(device=self.device, dtype=torch.int64)
        if ids.ndim == 1:
            ids = ids.unsqueeze(0).expand(n_q, -1)
        if ids.ndim != 2 or ids.shape[0] != n_q:
            raise ValueError(f"page_ids must be [n_cand] or [n_q={n_q}, n_cand], got {tuple(ids.shape)}")
        ids = ids.contiguous()
        n_cand, t_max, map_rows = int(ids.shape[1]), max(lens, default=0), int(map_rows)
        if map_rows < 0:
            raise ValueError("map_rows must be >= 0")
        ts = torch.empty((n_q, n_cand, t_max), dtype=torch.float32, device=self.device)
        br = torch.empty((n_q, n_cand, t_max), dtype=torch.int32, device=self.device)
        sm = torch.empty((n_q, n_cand, t_max, map_rows), dtype=torch.float32, device=self.device) if map_rows else None
        if n_q == 0 or n_cand == 0:
            return ts, br, sm
        src, src_dtype = self._stage_rows(list(queries))
        with torch.cuda.device(self.device):
            self.h.check(
                nat.lib.b200ms_explain_device(self.h.ptr, _vp(src), src_dtype, nat.i32_array(lens), n_q, _vp(ids), n_cand,
                                              ctypes.c_float(self.i8_scale), ctypes.c_float(self.score_scale), _vp(ts),
                                              _vp(br), _vp(sm), map_rows, self._stream()),
                "b200ms_explain_device")
        return ts, br, sm

    # ------------------------------------------------------------------ diversifying results
    def mmr(self, cand_ids: torch.Tensor, cand_scores: torch.Tensor, q_lens: Sequence[int], k: int, lambda_mult: float,
            with_sims: bool = False):
        """Maximal marginal relevance over each query's candidate list (b200ms_mmr_device), asynchronous on torch's current
        stream.  cand_ids int64 / cand_scores float32 [n_q, n_cand] on the device, as a search or rerank returned them (-1 =
        unused slot); q_lens the queries' token counts (relevance is score / tokens).  Picks greedily: first the most
        relevant page, then each time the page maximising lambda_mult * relevance - (1 - lambda_mult) * (its largest
        page-to-page MaxSim against a page picked already, per row of its own).  k is capped at n_cand.

        Returns device tensors (page ids int64 [n_q, k] in pick order, their input scores float32 [n_q, k], counts int32
        [n_q]) and, with ``with_sims``, sims float32 [n_q, k, n_cand]: sims[q, i, j] = the similarity of slot j to pick i,
        for the slots still unpicked after pick i (-inf elsewhere).  Works on both tiers; a host-tier call whose candidate
        pages do not fit one staging round raises NativeError."""
        n_q = len(q_lens)
        if cand_ids.ndim != 2 or cand_ids.shape[0] != n_q:
            raise ValueError(f"cand_ids must be [n_q = {n_q}, n_cand], got {tuple(cand_ids.shape)}")
        n_cand, kk = _check_candidates(cand_ids, n_q, k, self.device, per_query=True)
        if (cand_scores.dtype != torch.float32 or tuple(cand_scores.shape) != tuple(cand_ids.shape)
                or not cand_scores.is_contiguous() or cand_scores.device != self.device):
            raise ValueError(f"cand_scores must be a contiguous float32 {list(cand_ids.shape)} tensor on {self.device}")
        if not 0.0 <= float(lambda_mult) <= 1.0:  # NaN fails too
            raise ValueError(f"lambda_mult must be in [0, 1], got {lambda_mult}")
        if int(k) < 1 or n_cand < 1:
            raise ValueError("k and n_cand must be >= 1")
        if any(int(t) < 0 for t in q_lens):
            raise ValueError("query lengths must be >= 0")
        ts, ti, tc = _topk_outputs(n_q, kk, self.device)
        sims = torch.empty((n_q, kk, n_cand), dtype=torch.float32, device=self.device) if with_sims else None
        self._attach()
        with torch.cuda.device(self.device):
            self.h.check(
                nat.lib.b200ms_mmr_device(self.h.ptr, _vp(cand_ids), _vp(cand_scores), n_cand, nat.i32_array(q_lens), n_q, kk,
                                          ctypes.c_float(lambda_mult), ctypes.c_float(self.score_scale), _vp(ti), _vp(ts),
                                          _vp(tc), _vp(sims), self._stream()),
                "b200ms_mmr_device")
        return (ti, ts, tc, sims) if with_sims else (ti, ts, tc)

    # ------------------------------------------------------------------ near-duplicate pages
    def _check_pairs(self, pair_a: torch.Tensor, pair_b: torch.Tensor) -> int:
        for t in (pair_a, pair_b):
            if t.dtype != torch.int64 or t.ndim != 1 or not t.is_contiguous() or t.device != self.device:
                raise ValueError(f"pair ids must be contiguous int64 1-D tensors on {self.device}")
        if pair_a.shape != pair_b.shape:
            raise ValueError(f"pair_a and pair_b differ in length: {pair_a.shape[0]} != {pair_b.shape[0]}")
        return int(pair_a.shape[0])

    def pair_maxsim(self, pair_a: torch.Tensor, pair_b: torch.Tensor) -> Tuple[torch.Tensor, torch.Tensor]:
        """Both directions of page-to-page MaxSim for each pair (b200ms_pair_maxsim_device), asynchronous on torch's current
        stream: sim_ab[i] = sim(pair_a[i] -> pair_b[i]), sim_ba[i] = sim(pair_b[i] -> pair_a[i]), each the sum over the
        first page's true rows of their best dot product with a row of the second, times score_scale, over the first
        page's row count -- mmr(..., with_sims=True)'s value for the same pair, bit for bit.  One tensor-core product per pair
        serves both directions.  An id outside [0, n_pages) gives NaN, a page without rows 0.  HBM tier only."""
        n = self._check_pairs(pair_a, pair_b)
        sab = torch.empty((n,), dtype=torch.float32, device=self.device)
        sba = torch.empty((n,), dtype=torch.float32, device=self.device)
        self._attach()
        with torch.cuda.device(self.device):
            self.h.check(nat.lib.b200ms_pair_maxsim_device(self.h.ptr, _vp(pair_a), _vp(pair_b), n,
                                                           ctypes.c_float(self.score_scale), _vp(sab), _vp(sba),
                                                           self._stream()), "b200ms_pair_maxsim_device")
        return sab, sba

    def duplicate_groups(self, pair_a: torch.Tensor, pair_b: torch.Tensor, sim_ab: torch.Tensor, sim_ba: torch.Tensor,
                         threshold: float, allow_mask_dev: Optional[torch.Tensor] = None) -> torch.Tensor:
        """Duplicate groups (b200ms_duplicate_groups_device), asynchronous on torch's current stream: a pair is an edge when
        min(sim_ab, sim_ba) >= threshold (a NaN never is) and the allow mask (uint32 page words, None = every page) has both
        pages; groups are the connected components of the edges.  Returns int64 [n_pages] on the device: every allowed
        page's smallest group member, -1 for a page the mask excludes.  No threshold has been measured on real pages: the
        caller chooses it on the scale of the sims (pair_maxsim)."""
        n = self._check_pairs(pair_a, pair_b)
        for t in (sim_ab, sim_ba):
            if t.dtype != torch.float32 or t.shape != (n,) or not t.is_contiguous() or t.device != self.device:
                raise ValueError(f"sims must be contiguous float32 [{n}] tensors on {self.device}")
        if not math.isfinite(float(threshold)):
            raise ValueError(f"threshold must be a finite number, got {threshold}")
        masks = _check_device_masks(allow_mask_dev, None, 1, self.n_pages, self.device)[0]
        labels = torch.empty((self.n_pages,), dtype=torch.int64, device=self.device)
        self._attach()
        with torch.cuda.device(self.device):
            self.h.check(nat.lib.b200ms_duplicate_groups_device(self.h.ptr, _vp(pair_a), _vp(pair_b), _vp(sim_ab),
                                                                _vp(sim_ba), n, ctypes.c_float(threshold), _vp(masks),
                                                                _vp(labels), self._stream()),
                         "b200ms_duplicate_groups_device")
        return labels

    def duplicate_candidates(self, src_pages, n_candidates: int, allow_mask_dev: Optional[torch.Tensor] = None,
                             batch: int = DUP_SOURCE_BATCH) -> Tuple[torch.Tensor, torch.Tensor]:
        """Candidate pairs for the source pages: each source's top n_candidates other pages by search_pages under the allow
        mask (uint32 page words, None = every page), sources in batches of ``batch``.  Returns canonical pairs
        (candidate_pairs): device int64 (pair_a, pair_b), pair_a < pair_b, unique, ordered by (a, b)."""
        ids = self._src_pages(src_pages)
        n_cand = _check_n_candidates(n_candidates)
        parts = []
        for i in range(0, len(ids), int(batch)):
            src = ids[i:i + int(batch)]
            _, ti, _ = self.search_pages(src, min(n_cand + 1, nat.MAX_K), allow_mask_dev)
            parts.append((src, ti))
        return candidate_pairs(parts, n_cand, self.device)

    # ------------------------------------------------------------------ multi-GPU (document shards, NCCL inside libb200ms)
    @staticmethod
    def comm_unique_id() -> bytes:
        """128-byte NCCL unique id (rank 0 creates it; ship it to every rank by any channel)."""
        buf = (ctypes.c_uint8 * 128)()
        rc = nat.lib.b200ms_comm_unique_id(buf)
        if rc != 0:
            msg = nat.lib.b200ms_last_error(None)
            raise nat.NativeError(f"b200ms_comm_unique_id failed ({rc}): {msg.decode() if msg else ''}")
        return bytes(buf)

    def comm_init(self, unique_id: bytes, rank: int, world: int):
        """Collective: create this handle's NCCL communicator (libb200ms dlopens libnccl; torch is not involved)."""
        if len(unique_id) != 128:
            raise ValueError("unique_id must be the 128 bytes of comm_unique_id()")
        buf = (ctypes.c_uint8 * 128).from_buffer_copy(unique_id)
        with torch.cuda.device(self.device):
            self.h.check(nat.lib.b200ms_comm_init(self.h.ptr, buf, int(rank), int(world)), "b200ms_comm_init")

    def bcast(self, t: torch.Tensor, root: int = 0):
        """ncclBroadcast of a contiguous device tensor in place (e.g. the query rows of a batch) on torch's current stream."""
        with torch.cuda.device(self.device):
            self.h.check(nat.lib.b200ms_bcast_device(self.h.ptr, _vp(t), t.numel() * t.element_size(), int(root), self._stream()),
                         "b200ms_bcast_device")
        return t

    def send(self, t: torch.Tensor, peer: int):
        """ncclSend of a contiguous device tensor to rank `peer` over the handle's communicator (torch's current stream)."""
        with torch.cuda.device(self.device):
            self.h.check(nat.lib.b200ms_send_device(self.h.ptr, _vp(t), t.numel() * t.element_size(), int(peer), self._stream()),
                         "b200ms_send_device")

    def recv(self, t: torch.Tensor, peer: int):
        with torch.cuda.device(self.device):
            self.h.check(nat.lib.b200ms_recv_device(self.h.ptr, _vp(t), t.numel() * t.element_size(), int(peer), self._stream()),
                         "b200ms_recv_device")
        return t

    def allgather_topk(self, xchg: torch.Tensor, n_q: int, k: int, out=None):
        """The one collective of the path for a caller-made local list: xchg = uint8 device buffer in the exchange layout
        ([n_q*k int64 global ids][n_q*k float32 scores]) -> merged (scores, ids, counts), identical on every rank."""
        ts, ti, tc = _topk_outputs(int(n_q), int(k), self.device, out)
        with torch.cuda.device(self.device):
            self.h.check(nat.lib.b200ms_allgather_topk(self.h.ptr, None, _vp(xchg), int(n_q), int(k), _vp(ts), _vp(ti), _vp(tc),
                                                       self._stream()), "b200ms_allgather_topk")
        return ts, ti, tc

    def sharded_search_begin(self, q_dev: torch.Tensor, q_lens: Sequence[int], k: int, id_base: int,
                             out: Tuple[torch.Tensor, torch.Tensor, torch.Tensor],
                             allow_masks_dev: Optional[torch.Tensor] = None, mask_index_dev: Optional[torch.Tensor] = None) -> int:
        """Enqueue local scan + top-k on torch's current stream and the all-gather + merge behind it on the handle's
        communication stream; returns a ticket.  The current stream does not wait for the other ranks."""
        n_q = len(q_lens)
        q_dtype = _check_queries(q_dev, q_lens, self.device)
        masks, n_masks, index = _check_device_masks(allow_masks_dev, mask_index_dev, n_q, self.n_pages, self.device)
        ts, ti, tc = _topk_outputs(n_q, int(k), self.device, out)
        self._attach()
        with torch.cuda.device(self.device):
            t = int(nat.lib.b200ms_sharded_search_begin(
                self.h.ptr, _vp(q_dev), q_dtype, nat.i32_array(q_lens), n_q, int(k), _vp(masks), n_masks, _vp(index),
                ctypes.c_float(self.i8_scale), ctypes.c_float(self.score_scale), int(id_base), _vp(ts), _vp(ti), _vp(tc),
                self._stream()))
        if t < 0:
            self.h.check(t, "b200ms_sharded_search_begin")
        return t

    def sharded_search_end(self, ticket: int):
        """Make torch's current stream wait for that ticket's merged result (in the buffers given to begin)."""
        with torch.cuda.device(self.device):
            self.h.check(nat.lib.b200ms_sharded_search_end(self.h.ptr, int(ticket), self._stream()), "b200ms_sharded_search_end")

    def sharded_search_host_begin(self, q_host: torch.Tensor, q_lens: Sequence[int], k: int, id_base: int) -> int:
        """Host-buffer form: q_host float32 [sum T,128] (pinned for an asynchronous copy); returns a ticket."""
        self._attach()
        t = int(nat.lib.b200ms_sharded_search_host_begin(
            self.h.ptr, ctypes.c_void_p(q_host.data_ptr()), nat.i32_array(q_lens), len(q_lens), int(k), None, 0, None,
            ctypes.c_float(self.i8_scale), ctypes.c_float(self.score_scale), int(id_base)))
        if t < 0:
            self.h.check(t, "b200ms_sharded_search_host_begin")
        return t

    def sharded_search_host_end(self, ticket: int, out_scores: torch.Tensor, out_ids: torch.Tensor, out_counts: torch.Tensor):
        """Blocks until the ticket's merged top-k is on the host; fills the three (host) tensors."""
        self.h.check(nat.lib.b200ms_sharded_search_host_end(self.h.ptr, int(ticket), ctypes.c_void_p(out_scores.data_ptr()),
                                                            ctypes.c_void_p(out_ids.data_ptr()),
                                                            ctypes.c_void_p(out_counts.data_ptr())),
                     "b200ms_sharded_search_host_end")

    def close(self):
        self._buf = None
        if self._block is not None:
            torch.cuda.synchronize(self.device)
            self._block.free()
            self._block = None
        self.h.close()
