"""Two-stage search with an asymmetric 1-bit first stage: full-precision queries against an HBM copy of the corpus' sign bits
(b200ms_sign_candidates_device), then the exact MaxSim rerank of the candidates (b200ms_rerank_batch_device).

A sign row costs 16 B per patch vector, 1/16 of a bf16 row, so HBM holds the signs of a host-resident corpus many times
its own size and every page of them is scanned exhaustively; only the candidates' rows cross PCIe.  The query keeps its
magnitudes (quantised to int8 in [-63, 63]), unlike the symmetric Hamming MaxSim that sign-packs the query too.

``SignTwoStageIndex`` is the sign first stage of ``two_stage.TwoStageSearch``, beside ``fde.TwoStageIndex``.
"""
from __future__ import annotations

import ctypes
from typing import Optional, Sequence, Tuple

import numpy as np
import torch

from . import _native as nat
from .index import DeviceBlock, MaxSimIndex, _check_device_masks, _check_queries, _compact_rows, _row_runs, _topk_outputs, _vp
from .two_stage import TwoStageSearch

# q8 = clamp(rint(x * scale), -63, 63) of the query's elements; README "Sign candidates" has the recall against the scale
# that chose it
DEFAULT_Q_SCALE = 127.0


class SignTwoStageIndex(TwoStageSearch):
    """MaxSimIndex (bf16 / int8 / fp8, either tier) + the sign rows of its packed rows in a growable HBM block.

    The sign rows mirror the packed corpus row for row (padding rows included) and are derived on the GPU from the packed
    values (b200ms_sign_rows): appends derive only the new pages, ``compact`` moves them with the patch rows' runs, and
    ``rebuild_from_index`` derives them all (a corpus loaded from a shard file)."""
    STAGE_TIMES = {"stage_queries_ms": (0, 1), "sign_candidates_ms": (1, 2)}

    def __init__(self, device: int = 0, dtype: str = "bf16", index: Optional[MaxSimIndex] = None, tier: str = "hbm",
                 q_scale: float = DEFAULT_Q_SCALE):
        super().__init__(index if index is not None else MaxSimIndex(device=device, dtype=dtype, tier=tier))
        if self.index.dtype == nat.B1:
            raise ValueError("sign candidates need a bf16, int8 or fp8 corpus: a 1-bit corpus has no more precise rows to rerank")
        if not (np.isfinite(q_scale) and q_scale > 0):
            raise ValueError("q_scale must be finite and > 0")
        self.q_scale = float(q_scale)
        self._block: Optional[DeviceBlock] = None  # owner of the memory self._S views
        self._S: Optional[torch.Tensor] = None     # uint8 [backed rows, 16]
        self._rows = 0                             # padded rows whose signs are in _S

    def sign_rows(self) -> torch.Tensor:
        """The sign rows as uint8 [n_rows_padded, 16] (a view of the block)."""
        if self._S is None or self._rows == 0:
            return torch.empty((0, 16), dtype=torch.uint8, device=self.device)
        return self._S[: self._rows]

    def _resize(self, rows: int) -> None:
        self._block = DeviceBlock.resized(self._block, self.index.h, self.device, rows * 16)
        self._S = self._block.rows(16)

    def _derive(self, first: int, n: int) -> None:
        """Signs of pages [first, first + n) of the attached corpus into their rows of the block (pages before `first` keep
        theirs)."""
        self.index._attach()
        r0, r1 = self.index.page_row_range(first, n)
        if r1 > (0 if self._S is None else self._S.shape[0]):
            self._resize(r1)
        if r1 > r0:
            with torch.cuda.device(self.device):
                self.index.h.check(nat.lib.b200ms_sign_rows(self.index.h.ptr, first, n, _vp(self._S[r0:]), self.index._stream()),
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

    def replay_done(self) -> None:
        self.rebuild_from_index()  # once, over every replayed segment: sign rows are not persisted

    def compact(self, keep: Sequence[int]) -> None:
        """Keep only pages `keep` (ascending old ids): the patch rows and the sign rows move down in place, run for run."""
        keep = [int(p) for p in keep]
        runs = _row_runs(self.index.page_lens, keep)
        self.index.compact(keep)
        new_rows = sum(b - a for a, b in runs)
        if self._S is not None:
            _compact_rows(self.index.h, self.device, self._S, 16, runs)
            self._resize(new_rows)
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

    _scan = candidates_device
