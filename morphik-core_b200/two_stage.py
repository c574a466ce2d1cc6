"""Two-stage search: a first stage (``fde.TwoStageIndex``, ``signs.SignTwoStageIndex``) picks candidate pages per query
from side data it appends, rebuilds and compacts with the corpus; ``TwoStageSearch`` reranks them by exact MaxSim."""
from __future__ import annotations

from typing import Dict, Optional, Sequence, Tuple

import numpy as np
import torch

from . import _native as nat
from .index import DUP_SOURCE_BATCH, MaxSimIndex, _check_device_masks, _check_n_candidates, _host_mask_to_device, candidate_pairs


def _host(t: torch.Tensor, shape: Tuple[int, ...], fill) -> np.ndarray:
    """Device results [n_q, kk, ...] -> host array of `shape` ([n_q, k, ...], k >= kk) and their dtype, `fill` past kk."""
    a = t.cpu().numpy()
    out = np.full(shape, fill, dtype=a.dtype)
    out[:, :a.shape[1]] = a
    return out


class TwoStageSearch:
    # last_timing_ms names of the first stage's windows: name -> (first event, last event) of search_device's events
    STAGE_TIMES: Dict[str, Tuple[int, int]] = {}

    def __init__(self, index: MaxSimIndex):
        self.index = index
        self.device = index.device
        self.last_timing_ms: Dict[str, float] = {}

    @property
    def n_pages(self) -> int:
        return self.index.n_pages

    # ------------------------------------------------------------------ what a first stage supplies
    def _encode(self, queries: Sequence, staged: Optional[Tuple[torch.Tensor, int, Sequence[int]]]):
        """The queries as the scan takes them (part of the query preparation window): here their staged rows.  `staged`:
        (rows, dtype code, lengths) when the caller staged them already for the rerank, else None."""
        return staged[0] if staged else self.index._stage_rows(list(queries))[0]

    def _scan(self, q, lens: Sequence[int], n_cand: int, mask: Optional[torch.Tensor],
              mask_index: Optional[torch.Tensor] = None):
        """Top n_cand pages per query among those `mask` (checked, one row for every query; with ``mask_index`` int32
        [n_q], a [n_masks, words] matrix and each query's row, -1 = unfiltered) allows: device tensors (scores float32
        [n_q, n_cand], page ids int64 [n_q, n_cand] (-1 padded), counts int32 [n_q])."""
        raise NotImplementedError

    def journal_rows(self, first: int, n: int):
        """What a journal segment persists of the first stage for pages [first, first + n); None: nothing."""
        return None

    def replay_segment(self, path: str) -> None:
        """Journal replay: the segment just loaded into the index had its first-stage rows persisted at `path`, if at all."""

    def replay_done(self) -> None:
        """Journal replay: every segment is loaded."""

    # ------------------------------------------------------------------ the two-stage search
    def _mask(self, allow_mask_dev: Optional[torch.Tensor], n_q: int) -> Optional[torch.Tensor]:
        return _check_device_masks(allow_mask_dev, None, n_q, self.n_pages, self.device)[0]

    def _prepare(self, queries: Sequence):
        """Stages the query rows once: (rows, lengths, the rows as the scan takes them)."""
        src, src_dtype = self.index._stage_rows(list(queries))
        lens = [int(q.shape[0]) for q in queries]
        return src, lens, self._encode(queries, (src, src_dtype, lens))

    def _n_cand(self, want: int) -> int:
        return int(min(want, nat.MAX_K, max(self.n_pages, 1)))

    def candidates(self, queries: Sequence, n_candidates: int, allow_mask_dev: Optional[torch.Tensor] = None):
        """First stage only: (candidate page ids int64 [n_q, n_candidates] (-1 padded), first-stage scores, counts) on the
        device.  allow_mask_dev: optional uint32 page bitmask (the doc_ids filter, applied BEFORE candidate selection like the
        reference's Turbopuffer filter, fast_multivector_store.py:527)."""
        mask = self._mask(allow_mask_dev, len(queries))
        q = self._encode(queries, None)  # no rerank follows: the rows are staged (at most) once, for the scan
        ts, ti, tc = self._scan(q, [int(x.shape[0]) for x in queries], int(min(n_candidates, nat.MAX_K)), mask)
        return ti, ts, tc

    def rerank(self, query, cand_ids: torch.Tensor, k: int):
        """Exact MaxSim of ONE query over the candidate pages (device int64 [n_cand], -1 = unused) -> top-k."""
        src, _ = self.index._stage_rows([query])
        return self.index.rerank(src, [int(query.shape[0])], cand_ids.contiguous(), k)

    def search_device(self, queries: Sequence, k: int, n_candidates: int = 1000, allow_mask_dev: Optional[torch.Tensor] = None,
                      id_base: int = 0):
        """Two-stage search, everything on the device and asynchronous: max(n_candidates, k) candidates per query (at most
        MAX_K) from ONE first-stage scan for the whole batch -> ONE batched rerank call (each query against its own list) ->
        top-k.  Returns device tensors (scores [n_q,kk], page ids + id_base [n_q,kk], counts [n_q]) and the CUDA events that
        bracket the stages: query preparation, candidate scan + top-k, rerank."""
        mask = self._mask(allow_mask_dev, len(queries))
        ev = [torch.cuda.Event(enable_timing=True) for _ in range(4)]
        ev[0].record()
        src, lens, q = self._prepare(queries)
        ev[1].record()
        _, ci, _ = self._scan(q, lens, self._n_cand(max(n_candidates, k)), mask)
        ev[2].record()
        ts, ti, tc = self.index.rerank_batch(src, lens, ci, k)
        if id_base:
            ti = torch.where(ti >= 0, ti + int(id_base), ti)
        ev[3].record()
        return ts, ti, tc, ev

    def stage_timing_ms(self, ev) -> Dict[str, float]:
        """Stage times of a finished search_device call from its events: the first stage's windows, maxsim_rerank_ms and,
        of the rerank, load_multivectors_ms (the host tier's PCIe gather; 0 in HBM) and rerank_scoring_ms -- the reference's
        stage names (fast_multivector_store.py:523,534,550,574)."""
        out = {name: ev[a].elapsed_time(ev[b]) for name, (a, b) in self.STAGE_TIMES.items()}
        rerank_ms = ev[2].elapsed_time(ev[3])
        gather = self.index.gather_stats() if self.index.tier == "host" else {"ms": 0.0, "bytes": 0, "unique_pages": 0}
        out.update(maxsim_rerank_ms=rerank_ms, load_multivectors_ms=gather["ms"], rerank_scoring_ms=rerank_ms - gather["ms"],
                   gather_bytes=gather["bytes"], gather_pages=gather["unique_pages"])
        return out

    def search(self, queries: Sequence, k: int, n_candidates: int = 1000, allow_mask: Optional[np.ndarray] = None):
        """Two-stage search with a host allow mask (uint32 words, restricting both stages); synchronous.  Returns host arrays
        (scores [n_q,k], page ids [n_q,k], counts [n_q]) and fills last_timing_ms (stage_timing_ms)."""
        n_q = len(queries)
        mask_dev = _host_mask_to_device(allow_mask, self.n_pages, self.device)
        ts, ti, tc, ev = self.search_device(queries, k, n_candidates, mask_dev)
        torch.cuda.synchronize(self.device)
        out = _host(ts, (n_q, k), -np.inf), _host(ti, (n_q, k), -1), tc.cpu().numpy().astype(np.int32)
        self.last_timing_ms = self.stage_timing_ms(ev)
        return out

    def search_pages_device(self, src_pages, k: int, n_candidates: int = 1000, allow_mask_dev: Optional[torch.Tensor] = None,
                            mask_index_dev: Optional[torch.Tensor] = None, id_base: int = 0):
        """search_device with stored pages as the queries: the first stage runs on each source page's rows, dequantised on
        the device (MaxSimIndex.page_rows), and MaxSimIndex.rerank_pages_batch reranks its candidates with the packed page
        query, so scores are MaxSimIndex.search_pages's.  Masks as search_pages, one row per source, in BOTH stages: a page
        a source may not return (the source itself, its document) never takes one of its candidate slots.  Returns as
        search_device."""
        ids = self.index._src_pages(src_pages)
        masks, _, index = _check_device_masks(allow_mask_dev, mask_index_dev, len(ids), self.n_pages, self.device)
        ev = [torch.cuda.Event(enable_timing=True) for _ in range(4)]
        ev[0].record()
        rows, lens = self.index.page_rows(ids)
        q = self._encode(None, (rows, nat.F32, lens))
        ev[1].record()
        if index is None:
            _, ci, _ = self._scan(q, lens, self._n_cand(max(n_candidates, k)), masks)
        else:
            _, ci, _ = self._scan(q, lens, self._n_cand(max(n_candidates, k)), masks, index)
        ev[2].record()
        ts, ti, tc = self.index.rerank_pages_batch(ids, ci, k, allow_mask_dev, mask_index_dev)
        if id_base:
            ti = torch.where(ti >= 0, ti + int(id_base), ti)
        ev[3].record()
        return ts, ti, tc, ev

    def search_pages(self, src_pages, k: int, n_candidates: int = 1000, allow_masks: Optional[np.ndarray] = None):
        """search_pages_device with host masks: ``allow_masks`` uint32 [n_src, words], one row per source, or None;
        synchronous.  Returns host arrays (scores [n_src,k], page ids [n_src,k], counts [n_src]) and fills last_timing_ms with
        search's stage names."""
        n_src = len(self.index._src_pages(src_pages))
        words = (self.n_pages + 31) // 32
        masks = index = None
        if allow_masks is not None:
            m = np.ascontiguousarray(allow_masks, dtype=np.uint32)
            if m.shape != (n_src, words):
                raise ValueError(f"allow_masks must be uint32 [{n_src}, {words}], got {m.shape}")
            masks = torch.from_numpy(m.view(np.int32)).to(self.device)
            index = torch.arange(n_src, dtype=torch.int32, device=self.device)
        ts, ti, tc, ev = self.search_pages_device(src_pages, k, n_candidates, masks, index)
        torch.cuda.synchronize(self.device)
        out = _host(ts, (n_src, k), -np.inf), _host(ti, (n_src, k), -1), tc.cpu().numpy().astype(np.int32)
        self.last_timing_ms = self.stage_timing_ms(ev)
        return out

    def search_examples_device(self, queries: Sequence, pages, ex_req: Sequence[int], ex_weights: Sequence[float], n_req: int,
                               k: int, n_candidates: int = 1000, allow_mask_dev: Optional[torch.Tensor] = None,
                               mask_index_dev: Optional[torch.Tensor] = None, id_base: int = 0):
        """MaxSimIndex.search_examples through the first stage: the query embeddings ``queries`` (host [T,128] arrays) and
        stored ``pages`` are the examples, in that order, with ``ex_req`` / ``ex_weights`` as there.  Only the POSITIVE
        examples pick candidates -- query embeddings through _encode, pages through their dequantised rows
        (MaxSimIndex.page_rows) -- each under its request's mask row, in one first-stage scan; a request's lists are joined
        by MaxSimIndex.union_candidates, and MaxSimIndex.rerank_examples_batch scores every example, negatives included,
        against that union.  Returns as search_device."""
        queries = list(queries)
        ev = [torch.cuda.Event(enable_timing=True) for _ in range(4)]
        ev[0].record()
        src = self.index._stage_rows(queries)[0] if queries else None
        _, q_lens, pages, req, w = self.index._examples(src, [int(q.shape[0]) for q in queries], pages, ex_req, ex_weights,
                                                        n_req)
        masks, _, index = self.index._request_masks(allow_mask_dev, mask_index_dev, int(n_req))
        if masks is not None and masks.ndim == 1:
            masks = masks.view(1, -1)
        n_qe = len(q_lens)
        pos = sorted((r, i) for i, (r, x) in enumerate(zip(req, w)) if x > 0)  # by request, then in example order
        q_off = np.concatenate([[0], np.cumsum(q_lens, dtype=np.int64)]) if n_qe else None
        pos_pages = [i - n_qe for _, i in pos if i >= n_qe]
        p_rows, p_lens = self.index.page_rows([pages[j] for j in pos_pages]) if pos_pages else (None, [])
        p_off = np.concatenate([[0], np.cumsum(p_lens, dtype=np.int64)])
        rows, lens, j = [], [], 0
        for _, i in pos:
            if i < n_qe:
                rows.append(src[int(q_off[i]):int(q_off[i + 1])].float())
                lens.append(q_lens[i])
            else:
                rows.append(p_rows[int(p_off[j]):int(p_off[j + 1])])
                lens.append(int(p_lens[j]))
                j += 1
        q = self._encode(None, (torch.cat(rows).contiguous(), nat.F32, lens))
        ev[1].record()
        n_cand = self._n_cand(max(n_candidates, k))
        if index is None:
            _, ci, _ = self._scan(q, lens, n_cand, masks)
        else:
            pos_index = index[torch.tensor([r for r, _ in pos], dtype=torch.int64, device=self.device)].contiguous()
            _, ci, _ = self._scan(q, lens, n_cand, masks, pos_index)
        counts = np.bincount([r for r, _ in pos], minlength=int(n_req))
        union = self.index.union_candidates(ci.contiguous(), np.concatenate([[0], np.cumsum(counts)]).tolist())
        ev[2].record()
        ts, ti, tc = self.index.rerank_examples_batch(src, q_lens, pages, req, w, n_req, union, k, masks, index)
        if id_base:
            ti = torch.where(ti >= 0, ti + int(id_base), ti)
        ev[3].record()
        return ts, ti, tc, ev

    def search_examples(self, queries: Sequence, pages, ex_req: Sequence[int], ex_weights: Sequence[float], n_req: int, k: int,
                        n_candidates: int = 1000, allow_masks: Optional[np.ndarray] = None):
        """search_examples_device with host masks: ``allow_masks`` uint32 [n_req, words], one row per request, or None;
        synchronous.  Returns host arrays (scores [n_req,k], page ids [n_req,k], counts [n_req]) and fills last_timing_ms
        with search's stage names."""
        n_req = int(n_req)
        words = (self.n_pages + 31) // 32
        masks = index = None
        if allow_masks is not None:
            m = np.ascontiguousarray(allow_masks, dtype=np.uint32)
            if m.shape != (n_req, words):
                raise ValueError(f"allow_masks must be uint32 [{n_req}, {words}], got {m.shape}")
            masks = torch.from_numpy(m.view(np.int32)).to(self.device)
            index = torch.arange(n_req, dtype=torch.int32, device=self.device)
        ts, ti, tc, ev = self.search_examples_device(queries, pages, ex_req, ex_weights, n_req, k, n_candidates, masks, index)
        torch.cuda.synchronize(self.device)
        out = _host(ts, (n_req, k), -np.inf), _host(ti, (n_req, k), -1), tc.cpu().numpy().astype(np.int32)
        self.last_timing_ms = self.stage_timing_ms(ev)
        return out

    def search_docs_device(self, queries: Sequence, k: int, per_doc: int, page_doc_dev: torch.Tensor, n_docs: int,
                           n_candidates: int = 1000, allow_mask_dev: Optional[torch.Tensor] = None):
        """Two-stage search grouped by document: max(n_candidates, k * per_doc) candidates per query (at most MAX_K), then
        MaxSimIndex.rerank_docs_batch over them.  Returns its four device tensors."""
        mask = self._mask(allow_mask_dev, len(queries))
        src, lens, q = self._prepare(queries)
        _, ci, _ = self._scan(q, lens, self._n_cand(max(n_candidates, k * per_doc)), mask)
        return self.index.rerank_docs_batch(src, lens, ci, k, per_doc, page_doc_dev, n_docs)

    def search_docs(self, queries: Sequence, k: int, per_doc: int, page_doc_dev: torch.Tensor, n_docs: int,
                    n_candidates: int = 1000, allow_mask: Optional[np.ndarray] = None):
        """search_docs_device with a host allow mask (uint32 words, restricting both stages); synchronous, returns host
        arrays (scores [n_q,k,per_doc], page ids [n_q,k,per_doc], pages per document [n_q,k], documents [n_q])."""
        mask_dev = _host_mask_to_device(allow_mask, self.n_pages, self.device)
        ts, ti, pc, dc = self.search_docs_device(queries, k, per_doc, page_doc_dev, n_docs, n_candidates, mask_dev)
        n_q = len(queries)
        return (_host(ts, (n_q, k, per_doc), -np.inf), _host(ti, (n_q, k, per_doc), -1), _host(pc, (n_q, k), 0),
                dc.cpu().numpy())

    def search_doc_maxsim(self, queries: Sequence, k: int, per_doc: int, page_doc_dev: torch.Tensor, n_docs: int,
                          n_candidates: int = 1000, allow_mask: Optional[np.ndarray] = None):
        """Document-level MaxSim through the first stage: max(n_candidates, k) candidate pages per query, then
        MaxSimIndex.rerank_doc_maxsim_batch scores every allowed page of their documents.  The host allow mask (uint32
        words) restricts both stages.  Synchronous; returns host arrays as MaxSimIndex.search_doc_maxsim."""
        mask_dev = _host_mask_to_device(allow_mask, self.n_pages, self.device)
        mask = self._mask(mask_dev, len(queries))
        src, lens, q = self._prepare(queries)
        _, ci, _ = self._scan(q, lens, self._n_cand(max(n_candidates, k)), mask)
        out = self.index.rerank_doc_maxsim_batch(src, lens, ci, k, per_doc, page_doc_dev, n_docs, allow_mask_dev=mask_dev)
        return tuple(t.cpu().numpy() for t in out)

    def duplicate_candidates(self, src_pages, n_candidates: int, allow_mask_dev: Optional[torch.Tensor] = None,
                             batch: int = DUP_SOURCE_BATCH) -> Tuple[torch.Tensor, torch.Tensor]:
        """Candidate pairs for the source pages from the first stage alone: each source's dequantised rows
        (MaxSimIndex.page_rows) go through the first-stage scan under the allow mask (uint32 page words, None = every page),
        and its first n_candidates other pages become pairs.  No rerank: MaxSimIndex.pair_maxsim scores the pairs.  Returns
        canonical pairs as MaxSimIndex.duplicate_candidates."""
        ids = self.index._src_pages(src_pages)
        n_cand = _check_n_candidates(n_candidates)
        parts = []
        for i in range(0, len(ids), int(batch)):
            src = ids[i:i + int(batch)]
            rows, lens = self.index.page_rows(src)
            q = self._encode(None, (rows, nat.F32, lens))
            _, ci, _ = self._scan(q, lens, self._n_cand(n_cand + 1), self._mask(allow_mask_dev, len(src)))
            parts.append((src, ci))
        return candidate_pairs(parts, n_cand, self.device)

    def explain(self, queries: Sequence, page_ids, map_rows: int = 0):
        """Per-token breakdown of the named pages' MaxSim (MaxSimIndex.explain): the pages a search returned are explained by
        the same exact scorer that ranked them."""
        return self.index.explain(queries, page_ids, map_rows)
