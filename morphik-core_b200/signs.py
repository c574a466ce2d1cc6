"""Two-stage search with an asymmetric 1-bit first stage: full-precision queries against an HBM copy of the corpus' sign bits
(b200ms_sign_candidates_device), then the exact MaxSim rerank of the candidates (b200ms_rerank_batch_device).

A sign row costs 16 B per patch vector, 1/16 of a bf16 row, so HBM holds the signs of a host-resident corpus many times
its own size and every page of them is scanned exhaustively; only the candidates' rows cross PCIe.  The query keeps its
magnitudes (quantised to int8 in [-63, 63]), unlike the symmetric Hamming MaxSim that sign-packs the query too.

``SignTwoStageIndex`` has the surface ``B200MultiVectorStore`` uses on ``fde.TwoStageIndex``.
"""
from __future__ import annotations

import ctypes
from typing import Dict, Optional, Sequence, Tuple

import numpy as np
import torch

from . import _native as nat
from .index import (DeviceBlock, MaxSimIndex, _check_device_masks, _check_queries, _host_mask_to_device, _padded_lens, _runs,
                    _topk_outputs, _vp)

# q8 = clamp(rint(x * scale), -63, 63) of the query's elements; README "Sign candidates" has the recall against the scale
# that chose it
DEFAULT_Q_SCALE = 127.0


class SignTwoStageIndex:
    """MaxSimIndex (bf16 / int8 / fp8, either tier) + the sign rows of its packed rows in a growable HBM block.

    The sign rows mirror the packed corpus row for row (padding rows included) and are derived on the GPU from the packed
    values (b200ms_sign_rows): appends derive only the new pages, ``compact`` moves them with the patch rows' runs, and
    ``rebuild_from_index`` derives them all (a corpus loaded from a shard file)."""

    def __init__(self, device: int = 0, dtype: str = "bf16", index: Optional[MaxSimIndex] = None, tier: str = "hbm",
                 q_scale: float = DEFAULT_Q_SCALE):
        self.index = index if index is not None else MaxSimIndex(device=device, dtype=dtype, tier=tier)
        if self.index.dtype == nat.B1:
            raise ValueError("sign candidates need a bf16, int8 or fp8 corpus: a 1-bit corpus has no more precise rows to rerank")
        if not (np.isfinite(q_scale) and q_scale > 0):
            raise ValueError("q_scale must be finite and > 0")
        self.q_scale = float(q_scale)
        self.device = self.index.device
        self._block: Optional[DeviceBlock] = None  # owner of the memory self._S views
        self._S: Optional[torch.Tensor] = None     # uint8 [backed bytes]: 16 B per padded row
        self._rows = 0                             # padded rows whose signs are in _S
        self.last_timing_ms: Dict[str, float] = {}

    @property
    def n_pages(self) -> int:
        return self.index.n_pages

    def sign_rows(self) -> torch.Tensor:
        """The sign rows as uint8 [n_rows_padded, 16] (a view of the block)."""
        if self._S is None or self._rows == 0:
            return torch.empty((0, 16), dtype=torch.uint8, device=self.device)
        return self._S[: self._rows * 16].view(self._rows, 16)

    def _resize(self, rows: int) -> None:
        if self._block is None:
            self._block = DeviceBlock(self.index.h, self.device)
        self._block.resize(rows * 16)
        self._S = self._block.tensor

    def _derive(self, first: int, n: int) -> None:
        """Signs of pages [first, first + n) of the attached corpus into their rows of the block (pages before `first` keep
        theirs)."""
        self.index._attach()
        r0, r1 = self.index.page_row_range(first, n)
        if r1 > (0 if self._S is None else self._S.numel() // 16):
            self._resize(r1)
        if r1 > r0:
            with torch.cuda.device(self.device):
                self.index.h.check(nat.lib.b200ms_sign_rows(self.index.h.ptr, first, n, _vp(self._S[r0 * 16:]),
                                                            self.index._stream()),
                                   "b200ms_sign_rows")
        self._rows = r1

    def add_pages(self, pages: Sequence) -> Tuple[int, int]:
        first, n = self.index.add_pages(pages)
        if n:
            self._derive(first, n)
        return first, n

    def adopt_packed(self, rows: torch.Tensor, page_lens: Sequence[int]) -> None:
        """Adopt an already packed device corpus (MaxSimIndex.adopt_packed) and derive its sign rows."""
        self.index.adopt_packed(rows, page_lens)
        self.rebuild_from_index()

    def rebuild_from_index(self) -> None:
        """(Re)derive the sign rows of every page of the index from its packed rows -- the path of ``store.load`` / ``open``."""
        self._rows = 0
        self._derive(0, self.index.n_pages)

    def compact(self, keep: Sequence[int]) -> None:
        """Keep only pages `keep` (ascending old ids): the patch rows and the sign rows move down in place, run for run."""
        keep = [int(p) for p in keep]
        pad = _padded_lens(self.index.page_lens)
        starts = np.concatenate([[0], np.cumsum(pad)]).astype(np.int64)
        runs = [(int(starts[a]), int(starts[b + 1])) for a, b in _runs(keep)]
        self.index.compact(keep)
        new_rows = sum(b - a for a, b in runs)
        if self._S is not None:
            run_start = np.array([a for a, _ in runs], dtype=np.int64)
            run_rows = np.array([b - a for a, b in runs], dtype=np.int64)
            with torch.cuda.device(self.device):
                self.index.h.check(
                    nat.lib.b200ms_compact_rows(self.index.h.ptr, _vp(self._S), 16, run_start.ctypes.data_as(nat.i64p),
                                                run_rows.ctypes.data_as(nat.i64p), len(runs), self.index._stream()),
                    "b200ms_compact_rows")
            self._resize(new_rows)  # the shrink waits for the compaction (the handle's calls are ordered)
        self._rows = new_rows

    def _attach(self) -> None:
        """Attach the corpus, then its sign rows (every b200ms_set_corpus* detaches them)."""
        self.index._attach()
        if self._rows != self.index.n_rows_padded:
            raise RuntimeError("sign rows out of step with the corpus: pages were added to the index behind this object")
        with torch.cuda.device(self.device):
            self.index.h.check(nat.lib.b200ms_set_sign_rows(self.index.h.ptr, _vp(self._S) if self._rows else None, self._rows,
                                                            self.index._stream()), "b200ms_set_sign_rows")

    def candidates_device(self, q_dev: torch.Tensor, q_lens: Sequence[int], n_cand: int,
                          allow_mask_dev: Optional[torch.Tensor] = None, mask_index_dev: Optional[torch.Tensor] = None):
        """First stage on device query rows ([sum T,128] float32|bfloat16): the top n_cand pages of every query by the
        asymmetric sign score, among the pages its mask allows (masks as MaxSimIndex.search_device).  Returns device tensors
        (scores float32 [n_q, n_cand] = S / q_scale, page ids int64 [n_q, n_cand] (-1 padded), counts int32 [n_q])."""
        n_q = len(q_lens)
        q_dtype = _check_queries(q_dev, q_lens, self.device)
        masks, n_masks, index = _check_device_masks(allow_mask_dev, mask_index_dev, n_q, self.n_pages, self.device)
        if masks is not None and index is None:  # one mask for every query: a one-row matrix
            index = torch.zeros((n_q,), dtype=torch.int32, device=self.device)
        ts, ti, tc = _topk_outputs(n_q, int(n_cand), self.device)
        self._attach()
        with torch.cuda.device(self.device):
            self.index.h.check(
                nat.lib.b200ms_sign_candidates_device(
                    self.index.h.ptr, _vp(q_dev), q_dtype, nat.i32_array(q_lens), n_q, int(n_cand), _vp(masks), n_masks,
                    _vp(index), ctypes.c_float(self.q_scale), ctypes.c_float(1.0 / self.q_scale), _vp(ts), _vp(ti), _vp(tc),
                    self.index._stream()),
                "b200ms_sign_candidates_device")
        return ts, ti, tc

    def candidates(self, queries: Sequence, n_candidates: int, allow_mask_dev: Optional[torch.Tensor] = None):
        """First stage only, as TwoStageIndex.candidates: (page ids int64 [n_q, n_candidates] (-1 padded), scores, counts)."""
        src, _ = self.index._stage_rows(list(queries))
        ts, ti, tc = self.candidates_device(src, [int(q.shape[0]) for q in queries], int(min(n_candidates, nat.MAX_K)),
                                            allow_mask_dev)
        return ti, ts, tc

    def _n_cand(self, want: int) -> int:
        return int(min(want, nat.MAX_K, max(self.n_pages, 1)))

    def search_device(self, queries: Sequence, k: int, n_candidates: int = 1000, allow_mask_dev: Optional[torch.Tensor] = None,
                      id_base: int = 0):
        """Two-stage search on the device, asynchronous: sign candidates (max(n_candidates, k), at most MAX_K, per query) ->
        ONE batched rerank (each query against its own list) -> top-k.  Returns (scores [n_q,kk], page ids + id_base
        [n_q,kk], counts [n_q]) and the CUDA events that bracket the stages (staging, candidates, rerank)."""
        ev = [torch.cuda.Event(enable_timing=True) for _ in range(4)]
        ev[0].record()
        src, _ = self.index._stage_rows(list(queries))
        lens = [int(q.shape[0]) for q in queries]
        ev[1].record()
        _, ci, _ = self.candidates_device(src, lens, self._n_cand(max(n_candidates, k)), allow_mask_dev)
        ev[2].record()
        ts, ti, tc = self.index.rerank_batch(src, lens, ci, k)
        if id_base:
            ti = torch.where(ti >= 0, ti + int(id_base), ti)
        ev[3].record()
        return ts, ti, tc, ev

    def search(self, queries: Sequence, k: int, n_candidates: int = 1000, allow_mask: Optional[np.ndarray] = None):
        """Two-stage search with a host allow mask (uint32 words, restricting both stages); synchronous.  Returns host arrays
        (scores [n_q,k], page ids [n_q,k], counts [n_q]) and fills last_timing_ms with the stage split: sign_candidates_ms,
        maxsim_rerank_ms and, of the rerank, load_multivectors_ms (the host tier's PCIe gather; 0 in HBM) and
        rerank_scoring_ms."""
        n_q = len(queries)
        mask_dev = _host_mask_to_device(allow_mask, self.n_pages, self.device)
        ts, ti, tc, ev = self.search_device(queries, k, n_candidates, mask_dev)
        torch.cuda.synchronize(self.device)
        kk = ts.shape[1]
        out_s = np.full((n_q, k), -np.inf, dtype=np.float32)
        out_i = np.full((n_q, k), -1, dtype=np.int64)
        out_s[:, :kk], out_i[:, :kk] = ts.cpu().numpy(), ti.cpu().numpy()
        out_c = tc.cpu().numpy().astype(np.int32)
        rerank_ms = ev[2].elapsed_time(ev[3])
        gather = self.index.gather_stats() if self.index.tier == "host" else {"ms": 0.0, "bytes": 0, "unique_pages": 0}
        self.last_timing_ms = {"stage_queries_ms": ev[0].elapsed_time(ev[1]), "sign_candidates_ms": ev[1].elapsed_time(ev[2]),
                               "maxsim_rerank_ms": rerank_ms, "load_multivectors_ms": gather["ms"],
                               "rerank_scoring_ms": rerank_ms - gather["ms"], "gather_bytes": gather["bytes"],
                               "gather_pages": gather["unique_pages"]}
        return out_s, out_i, out_c

    def search_docs_device(self, queries: Sequence, k: int, per_doc: int, page_doc_dev: torch.Tensor, n_docs: int,
                           n_candidates: int = 1000, allow_mask_dev: Optional[torch.Tensor] = None):
        """Two-stage search grouped by document: max(n_candidates, k * per_doc) sign candidates per query (at most MAX_K),
        then MaxSimIndex.rerank_docs_batch over them.  Returns its four device tensors."""
        src, _ = self.index._stage_rows(list(queries))
        lens = [int(q.shape[0]) for q in queries]
        _, ci, _ = self.candidates_device(src, lens, self._n_cand(max(n_candidates, k * per_doc)), allow_mask_dev)
        return self.index.rerank_docs_batch(src, lens, ci, k, per_doc, page_doc_dev, n_docs)

    def search_docs(self, queries: Sequence, k: int, per_doc: int, page_doc_dev: torch.Tensor, n_docs: int,
                    n_candidates: int = 1000, allow_mask: Optional[np.ndarray] = None):
        """search_docs_device with a host allow mask (restricting both stages); synchronous, host arrays as
        TwoStageIndex.search_docs."""
        mask_dev = _host_mask_to_device(allow_mask, self.n_pages, self.device)
        ts, ti, pc, dc = self.search_docs_device(queries, k, per_doc, page_doc_dev, n_docs, n_candidates, mask_dev)
        n_q, kk = len(queries), ts.shape[1]
        out_s = np.full((n_q, k, per_doc), -np.inf, dtype=np.float32)
        out_i = np.full((n_q, k, per_doc), -1, dtype=np.int64)
        out_pc = np.zeros((n_q, k), dtype=np.int32)
        out_s[:, :kk], out_i[:, :kk], out_pc[:, :kk] = ts.cpu().numpy(), ti.cpu().numpy(), pc.cpu().numpy()
        return out_s, out_i, out_pc, dc.cpu().numpy()

    def explain(self, queries: Sequence, page_ids, map_rows: int = 0):
        """Per-token breakdown of the named pages' exact MaxSim (MaxSimIndex.explain)."""
        return self.index.explain(queries, page_ids, map_rows)
