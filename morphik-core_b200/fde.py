"""Fixed-dimensional encodings (MUVERA FDE) + two-stage search: FDE candidate scan -> exact MaxSim rerank.

API mirror of the reference's ``fixed_dimensional_encoding`` extension module as Morphik uses it
(core/vector_store/fast_multivector_store.py:325-331, 447-449, 521):

    cfg = FixedDimensionalEncodingConfig(dimension=128, num_repetitions=20, num_simhash_projections=5,
                                         projection_dimension=16, projection_type="AMS_SKETCH")
    q_fde = generate_query_encoding(q, cfg)        # np.ndarray [n,128] -> np.float32 [10240]
    d_fde = generate_document_encoding(p, cfg)

and ``TwoStageIndex``, which replaces stages 1-4 of FastMultiVectorStore.query_similar (:521-557): the query FDE, the
Turbopuffer ANN over document FDEs (cosine distance, ``top_k = min(10*k, 75)`` there; any candidate count here), the
gather of candidate multivectors and the MaxSim rerank -- all on the GPU, with the multivectors already resident.

PARITY NOTE (SURVEY F2): the extension's C++ sources are not in the reference snapshot, so the exact random streams of
the upstream implementation (std::mt19937 based) cannot be reproduced or checked here.  The construction (SimHash
partitions with Gray-code index, AMS sketch, SUM for queries / AVERAGE for documents, empty partitions zero or -- with
``fill_empty_partitions`` -- the projection of the nearest point, optional final count-sketch projection) follows the
published algorithm; by default the matrices come from ``numpy.random.default_rng(seed + repetition)``, so FDEs produced
here are self-consistent (query and document sides share the matrices) but NOT interchangeable with vectors already
stored in a Turbopuffer namespace by the reference.

LOADING UPSTREAM MATRICES: the random matrices are INPUTS of the C-ABI (``b200ms_fde_configure_ex``).  A deployment that
must stay interchangeable with vectors written by the reference dumps the extension's matrices once (SimHash Gaussian
[R,128,K], AMS bucket index / sign [R,128], and for ``final_projection_dimension`` the count-sketch index / sign
[R*2^K*P]) and passes them through ``FdeMatrices`` / ``matrices_from_npz`` -- every consumer below takes an optional
``matrices`` argument.  The encoder then reproduces upstream bit for bit up to fp32 summation order.
"""
from __future__ import annotations

import ctypes
import os
import threading
from dataclasses import dataclass
from typing import Dict, Optional, Sequence, Tuple

import numpy as np
import torch

from . import _native as nat
from .index import DeviceBlock, MaxSimIndex, _compact_rows, _runs, _topk_outputs, _vp
from .two_stage import TwoStageSearch


@dataclass(frozen=True)
class FixedDimensionalEncodingConfig:
    """Field names follow the upstream config message the reference fills at fast_multivector_store.py:325-331 (it sets
    only the first five; ``fill_empty_partitions`` and ``final_projection_dimension`` stay at their defaults there)."""
    dimension: int = 128
    num_repetitions: int = 20
    num_simhash_projections: int = 5
    projection_dimension: int = 16
    projection_type: str = "AMS_SKETCH"
    seed: int = 1
    fill_empty_partitions: bool = False
    final_projection_dimension: int = 0  # > 0: count-sketch the whole encoding down to this many dims

    @property
    def num_partitions(self) -> int:
        return 1 << self.num_simhash_projections

    @property
    def inner_dimension(self) -> int:
        return self.num_repetitions * self.num_partitions * self.projection_dimension

    @property
    def fde_dimension(self) -> int:
        return self.final_projection_dimension if self.final_projection_dimension > 0 else self.inner_dimension

    @property
    def scale(self) -> float:
        return 1.0 / float(np.sqrt(self.projection_dimension))

    def validate(self) -> None:
        if self.dimension != nat.DIM:
            raise ValueError(f"dimension must be {nat.DIM}")
        if self.projection_type != "AMS_SKETCH":
            raise ValueError("only projection_type='AMS_SKETCH' (the reference's setting) is implemented")
        if self.final_projection_dimension < 0 or self.final_projection_dimension % 8:
            raise ValueError("final_projection_dimension must be 0 or a positive multiple of 8")


@dataclass(frozen=True)
class FdeMatrices:
    """The random matrices of one configuration -- generated here (``fde_matrices_full``) or dumped from the upstream
    extension (``matrices_from_npz``)."""
    simhash: np.ndarray      # float32 [R,128,K] Gaussian SimHash projections
    ams_index: np.ndarray    # int32   [R,128]   AMS sketch: bucket of every input dim, in [0, projection_dimension)
    ams_sign: np.ndarray     # float32 [R,128]   +-1
    final_index: Optional[np.ndarray] = None  # int32   [inner_dimension] final count sketch: output dim of every entry
    final_sign: Optional[np.ndarray] = None   # float32 [inner_dimension] +-1


def fde_matrices_full(cfg: FixedDimensionalEncodingConfig) -> FdeMatrices:
    cfg.validate()
    R, K, P = cfg.num_repetitions, cfg.num_simhash_projections, cfg.projection_dimension
    simhash = np.empty((R, cfg.dimension, K), dtype=np.float32)
    ams_index = np.empty((R, cfg.dimension), dtype=np.int32)
    ams_sign = np.empty((R, cfg.dimension), dtype=np.float32)
    for r in range(R):
        rng = np.random.default_rng(cfg.seed + r)
        simhash[r] = rng.standard_normal((cfg.dimension, K)).astype(np.float32)
        ams_index[r] = rng.integers(0, P, size=cfg.dimension).astype(np.int32)
        ams_sign[r] = np.where(rng.integers(0, 2, size=cfg.dimension) == 1, 1.0, -1.0).astype(np.float32)
    fi = fs = None
    if cfg.final_projection_dimension > 0:
        rng = np.random.default_rng(cfg.seed + 1_000_003)
        fi = rng.integers(0, cfg.final_projection_dimension, size=cfg.inner_dimension).astype(np.int32)
        fs = np.where(rng.integers(0, 2, size=cfg.inner_dimension) == 1, 1.0, -1.0).astype(np.float32)
    return FdeMatrices(simhash, ams_index, ams_sign, fi, fs)


def fde_matrices(cfg: FixedDimensionalEncodingConfig) -> Tuple[np.ndarray, np.ndarray, np.ndarray]:
    """(simhash [R,128,K] float32 Gaussian, ams_index [R,128] int32 in [0,proj), ams_sign [R,128] float32 +-1)."""
    m = fde_matrices_full(cfg)
    return m.simhash, m.ams_index, m.ams_sign


def matrices_from_npz(path: str) -> FdeMatrices:
    """Load matrices dumped from the upstream ``fixed_dimensional_encoding`` extension (arrays ``simhash``, ``ams_index``,
    ``ams_sign`` and optionally ``final_index`` / ``final_sign``) so that encodings match vectors the reference stored."""
    z = np.load(path)
    return FdeMatrices(np.ascontiguousarray(z["simhash"], np.float32), np.ascontiguousarray(z["ams_index"], np.int32),
                       np.ascontiguousarray(z["ams_sign"], np.float32),
                       np.ascontiguousarray(z["final_index"], np.int32) if "final_index" in z else None,
                       np.ascontiguousarray(z["final_sign"], np.float32) if "final_sign" in z else None)


def configure_handle(index: MaxSimIndex, cfg: FixedDimensionalEncodingConfig, matrices: Optional[FdeMatrices] = None) -> None:
    cfg.validate()
    m = matrices or fde_matrices_full(cfg)
    R, K, P = cfg.num_repetitions, cfg.num_simhash_projections, cfg.projection_dimension
    if m.simhash.shape != (R, cfg.dimension, K) or m.ams_index.shape != (R, cfg.dimension) or m.ams_sign.shape != (R, cfg.dimension):
        raise ValueError("FDE matrices do not match the configuration")
    fd = cfg.final_projection_dimension
    if fd > 0 and (m.final_index is None or m.final_sign is None or m.final_index.shape != (cfg.inner_dimension,)):
        raise ValueError("final_projection_dimension needs final_index / final_sign of inner_dimension entries")
    vp = lambda a: None if a is None else np.ascontiguousarray(a).ctypes.data_as(ctypes.c_void_p)  # noqa: E731
    sh, ai, sg = (np.ascontiguousarray(m.simhash, np.float32), np.ascontiguousarray(m.ams_index, np.int32),
                  np.ascontiguousarray(m.ams_sign, np.float32))
    fi = None if fd == 0 else np.ascontiguousarray(m.final_index, np.int32)
    fs = None if fd == 0 else np.ascontiguousarray(m.final_sign, np.float32)
    index.h.check(
        nat.lib.b200ms_fde_configure_ex(index.h.ptr, R, K, P, ctypes.c_float(cfg.scale), vp(sh), vp(ai), vp(sg),
                                        int(cfg.fill_empty_partitions), int(fd), vp(fi), vp(fs)),
        "b200ms_fde_configure_ex")


def encode_rows(index: MaxSimIndex, src: torch.Tensor, src_dtype: int, lens: Sequence[int], is_document: bool,
                fde_dim: int) -> torch.Tensor:
    """FDEs of staged ragged items (``src`` [>= sum(lens), 128] on the device, item i = the next lens[i] rows) -> float32
    device tensor [len(lens), fde_dim] (one kernel launch per 65535 items)."""
    out = torch.empty((len(lens), fde_dim), dtype=torch.float32, device=index.device)
    step, row0 = 65535, 0
    for i0 in range(0, len(lens), step):
        part = [int(n) for n in lens[i0:i0 + step]]
        with torch.cuda.device(index.device):
            index.h.check(
                nat.lib.b200ms_fde_encode(index.h.ptr, _vp(src[row0:]), src_dtype, nat.i32_array(part), len(part),
                                          int(is_document), _vp(out[i0:i0 + len(part)]), index._stream()),
                "b200ms_fde_encode")
        row0 += sum(part)
    return out


def encode_items(index: MaxSimIndex, items: Sequence, is_document: bool, fde_dim: int) -> torch.Tensor:
    """FDEs of ragged [n_i,128] items -> float32 device tensor [len(items), fde_dim]."""
    src, src_dtype = index._stage_rows(list(items))
    return encode_rows(index, src, src_dtype, [int(x.shape[0]) for x in items], is_document, fde_dim)


# ------------------------------------------------------------------ module-level API (drop-in for the extension module)
_default_lock = threading.Lock()
_default_encoders: Dict[Tuple[int, FixedDimensionalEncodingConfig], MaxSimIndex] = {}


def _encoder(cfg: FixedDimensionalEncodingConfig, device: int = 0) -> MaxSimIndex:
    with _default_lock:
        key = (device, cfg)
        if key not in _default_encoders:
            idx = MaxSimIndex(device=device, dtype="bf16")  # only its handle/stream are used
            configure_handle(idx, cfg)
            _default_encoders[key] = idx
        return _default_encoders[key]


def generate_query_encoding(point_cloud, config: FixedDimensionalEncodingConfig, device: int = 0) -> np.ndarray:
    """fde.generate_query_encoding(np.ndarray [n,128], cfg) -> np.float32 [fde_dimension] (fast_multivector_store.py:521)."""
    x = np.ascontiguousarray(np.asarray(point_cloud, dtype=np.float32).reshape(-1, nat.DIM))
    idx = _encoder(config, device)
    return encode_items(idx, [x], False, config.fde_dimension)[0].cpu().numpy()


def generate_document_encoding(point_cloud, config: FixedDimensionalEncodingConfig, device: int = 0) -> np.ndarray:
    """fde.generate_document_encoding(np.ndarray [n,128], cfg) (fast_multivector_store.py:447-449)."""
    x = np.ascontiguousarray(np.asarray(point_cloud, dtype=np.float32).reshape(-1, nat.DIM))
    idx = _encoder(config, device)
    return encode_items(idx, [x], True, config.fde_dimension)[0].cpu().numpy()


# ------------------------------------------------------------------ two-stage index
class TwoStageIndex(TwoStageSearch):
    """MaxSimIndex + a dense FDE matrix [N, fde_dim] bf16 with per-row inverse norms.

    search(): query FDE (device) -> exhaustive cosine scan of the FDE matrix (HBM-bound, 2*fde_dim bytes per page) -> top
    ``n_candidates`` per query -> exact MaxSim over those pages only (TwoStageSearch) -> top-k.
    """
    STAGE_TIMES = {"encode_query_ms": (0, 1), "ns_query_ms": (1, 2), "fde_candidates_ms": (0, 2)}

    def __init__(self, device: int = 0, dtype: str = "bf16", config: Optional[FixedDimensionalEncodingConfig] = None,
                 matrices: Optional[FdeMatrices] = None, index: Optional[MaxSimIndex] = None, tier: str = "hbm"):
        """tier="host": the patch rows live in pinned host memory (MaxSimIndex tier "host") and every search gathers only
        its candidate pages over PCIe; the FDE matrix stays in HBM either way."""
        super().__init__(index if index is not None else MaxSimIndex(device=device, dtype=dtype, tier=tier))
        self.cfg = config or FixedDimensionalEncodingConfig()
        configure_handle(self.index, self.cfg, matrices)
        self.fde_dim = self.cfg.fde_dimension
        self._Fblock: Optional[DeviceBlock] = None  # owner of the memory self._F views
        self._F: Optional[torch.Tensor] = None  # bf16 [cap, fde_dim]
        self._inv: Optional[torch.Tensor] = None  # float32 [cap]
        self._n = 0

    @property
    def n_pages(self) -> int:
        return self._n

    def _grow(self, need: int) -> None:
        cap = 0 if self._F is None else self._F.shape[0]
        if need <= cap:
            return
        self._resize(need)

    def _resize(self, rows: int) -> None:
        """Back `rows` FDE rows (rounded up to whole chunks) of the matrix's block -- no copy of the matrix, as for the
        patch rows (MaxSimIndex._resize_block); _F is a view of the block.  The inverse norms (4 bytes per page) are a
        torch tensor of the same capacity and are copied."""
        self._Fblock = DeviceBlock.resized(self._Fblock, self.index.h, self.device, rows * 2 * self.fde_dim)
        F = self._Fblock.rows(2 * self.fde_dim)
        if F is None:
            self._F = self._inv = None
            return
        self._F = F.view(torch.bfloat16)
        inv = torch.empty((F.shape[0],), dtype=torch.float32, device=self.device)
        if self._inv is not None:
            n = min(self._n, F.shape[0])
            inv[:n].copy_(self._inv[:n])
        self._inv = inv

    def add_pages(self, pages: Sequence) -> Tuple[int, int]:
        first, n = self.index.add_pages(pages)
        if n == 0:
            return first, 0
        fde = encode_items(self.index, list(pages), True, self.fde_dim)
        self._grow(self._n + n)
        with torch.cuda.device(self.device):
            self.index.h.check(
                nat.lib.b200ms_fde_finalize(self.index.h.ptr, _vp(fde), n, _vp(self._F[self._n:]), _vp(self._inv[self._n:]),
                                            self.index._stream()),
                "b200ms_fde_finalize")
        self._n += n
        return first, n

    def adopt_packed(self, rows: torch.Tensor, page_lens: Sequence[int], batch_pages: int = 16384) -> None:
        """Adopt an already packed bf16 device corpus (see MaxSimIndex.adopt_packed) and build its FDE matrix from the packed
        rows directly.  Requires every page length to be a multiple of 32 (no padding rows inside the packed buffer)."""
        lens = [int(x) for x in page_lens]
        if self.index.dtype != nat.BF16 or any(n % 32 for n in lens):
            raise ValueError("adopt_packed needs a bf16 corpus whose page lengths are multiples of 32")
        self.index.adopt_packed(rows, lens)
        n = len(lens)
        self._grow(n)
        flat = rows.view(torch.uint8).reshape(-1)
        tmp = torch.empty((min(batch_pages, max(n, 1)), self.fde_dim), dtype=torch.float32, device=self.device)
        row0 = 0
        with torch.cuda.device(self.device):
            for i0 in range(0, n, batch_pages):
                part = lens[i0:i0 + batch_pages]
                src = flat[row0 * 256:]
                self.index.h.check(
                    nat.lib.b200ms_fde_encode(self.index.h.ptr, _vp(src), nat.BF16, nat.i32_array(part), len(part), 1, _vp(tmp),
                                              self.index._stream()), "b200ms_fde_encode")
                self.index.h.check(
                    nat.lib.b200ms_fde_finalize(self.index.h.ptr, _vp(tmp), len(part), _vp(self._F[i0:]), _vp(self._inv[i0:]),
                                                self.index._stream()), "b200ms_fde_finalize")
                row0 += sum(part)
        self._n = n

    def rebuild_from_index(self, batch_pages: int = 16384) -> None:
        """(Re)build the FDE matrix for every page of the attached bf16 corpus from its packed rows
        (b200ms_fde_encode_corpus) -- the path of ``store.load(..., fde_candidates=N)`` and of a journal replay."""
        if self.index.dtype != nat.BF16:
            raise ValueError("rebuilding FDEs from packed rows needs a bf16 corpus (other dtypes persist their FDE rows)")
        self.index._attach()
        n = self.index.n_pages
        self._n = 0
        self._grow(n)
        tmp = torch.empty((min(batch_pages, max(n, 1)), self.fde_dim), dtype=torch.float32, device=self.device)
        with torch.cuda.device(self.device):
            for i0 in range(0, n, batch_pages):
                m = min(batch_pages, n - i0)
                self.index.h.check(nat.lib.b200ms_fde_encode_corpus(self.index.h.ptr, i0, m, _vp(tmp), self.index._stream()),
                                   "b200ms_fde_encode_corpus")
                self.index.h.check(nat.lib.b200ms_fde_finalize(self.index.h.ptr, _vp(tmp), m, _vp(self._F[i0:]),
                                                               _vp(self._inv[i0:]), self.index._stream()), "b200ms_fde_finalize")
        self._n = n

    def fde_rows(self, first: int = 0, n: Optional[int] = None) -> Tuple[torch.Tensor, torch.Tensor]:
        """(bf16 [n, fde_dim], inv_norm float32 [n]) views of pages [first, first+n) -- what a journal segment persists."""
        n = self._n - first if n is None else n
        return self._F[first:first + n], self._inv[first:first + n]

    def append_fde_rows(self, rows: torch.Tensor, inv: torch.Tensor) -> None:
        """Adopt persisted FDE rows for pages already appended to the MaxSim corpus (journal replay)."""
        n = int(rows.shape[0])
        self._grow(self._n + n)
        self._F[self._n:self._n + n].copy_(rows.to(self.device))
        self._inv[self._n:self._n + n].copy_(inv.to(self.device))
        self._n += n

    def fde_scores(self, q_fde: torch.Tensor) -> torch.Tensor:
        """[n_q, fde_dim] float32 device -> cosine-ranking scores [n_q, ld] (ld >= n_pages)."""
        n_q = q_fde.shape[0]
        ld = max((self._n + 31) // 32 * 32, 32)
        scores = torch.empty((n_q, ld), dtype=torch.float32, device=self.device)
        with torch.cuda.device(self.device):
            self.index.h.check(
                nat.lib.b200ms_fde_scan(self.index.h.ptr, _vp(self._F), _vp(self._inv), self._n, _vp(q_fde.contiguous()), n_q,
                                        _vp(scores), ld, self.index._stream()),
                "b200ms_fde_scan")
        return scores

    def compact(self, keep: Sequence[int]) -> None:
        """Keep only pages `keep` (ascending old ids) in both the patch corpus and the FDE matrix, each in place."""
        keep = [int(p) for p in keep]
        self.index.compact(keep)
        if self._F is not None:
            keep_t = torch.as_tensor(keep, dtype=torch.int64, device=self.device)
            self._inv[: len(keep)] = self._inv.index_select(0, keep_t)
            _compact_rows(self.index.h, self.device, self._F, 2 * self.fde_dim, [(a, b + 1) for a, b in _runs(keep)])
            self._n = len(keep)
            self._resize(len(keep))
        self._n = len(keep)

    journal_rows = fde_rows

    def replay_segment(self, path: str) -> None:
        if os.path.exists(path):
            blob = torch.load(path)
            self.append_fde_rows(blob["rows"].view(torch.bfloat16), blob["inv"])
        else:
            self.rebuild_from_index()

    def _encode(self, queries: Sequence, staged) -> torch.Tensor:
        if staged is None:
            return encode_items(self.index, list(queries), False, self.fde_dim)
        return encode_rows(self.index, *staged, False, self.fde_dim)

    def _scan(self, q_fde: torch.Tensor, lens: Sequence[int], kc: int, mask: Optional[torch.Tensor],
              mask_index: Optional[torch.Tensor] = None):
        """Scan of the FDE matrix for query FDEs [n_q, fde_dim] -> top kc pages per query among those `mask` (already
        checked) allows: (scores, page ids, counts) on the device.  With ``mask_index`` (int32 [n_q], -1 = unfiltered),
        `mask` is a [n_masks, words] matrix and query q keeps to its row (b200ms_topk_masked)."""
        n_q = q_fde.shape[0]
        scores = self.fde_scores(q_fde)
        ts, ti, tc = _topk_outputs(n_q, kc, self.device)
        goff = nat.i32_array(list(range(n_q + 1)))
        with torch.cuda.device(self.device):
            if mask_index is not None:
                self.index.h.check(
                    nat.lib.b200ms_topk_masked(self.index.h.ptr, _vp(scores), nat.F32, self._n, scores.shape[1], goff, n_q,
                                               _vp(mask), int(mask.shape[0]), _vp(mask_index), kc, ctypes.c_float(1.0), 0,
                                               _vp(ts), _vp(ti), _vp(tc), self.index._stream()),
                    "b200ms_topk_masked(fde)")
                return ts, ti, tc
            self.index.h.check(
                nat.lib.b200ms_topk(self.index.h.ptr, _vp(scores), nat.F32, self._n, scores.shape[1], goff, n_q, _vp(mask), kc,
                                    ctypes.c_float(1.0), 0, _vp(ts), _vp(ti), _vp(tc), self.index._stream()),
                "b200ms_topk(fde)")
        return ts, ti, tc

