"""PageCatalog -- host-side bookkeeping next to the device corpus (pure Python/numpy; no CUDA).

The device only knows integer page ids.  Everything the reference keeps in relational columns next to the embeddings
(``document_id``, ``chunk_number``, ``content``, ``chunk_metadata`` of ``multi_vector_embeddings``,
core/vector_store/multi_vector_store.py:240-251) lives here, together with:
  * the ``WHERE document_id IN (...)`` filter (multi_vector_store.py:752-757;
    ``filters=("document_id","In",doc_ids)`` fast_multivector_store.py:527) turned into a per-page allow mask,
  * ``DELETE FROM multi_vector_embeddings WHERE document_id = ...`` (multi_vector_store.py:929-933) as tombstones
    plus a compaction plan.
"""
from __future__ import annotations

from collections import OrderedDict
from dataclasses import dataclass, field
from typing import Any, Dict, Iterable, List, Optional, Sequence, Tuple

import numpy as np


@dataclass
class PageRecord:
    document_id: str
    chunk_number: int
    content: str
    metadata: Dict[str, Any] = field(default_factory=dict)
    app_id: Optional[str] = None
    n_rows: int = 0


class PageCatalog:
    def __init__(self) -> None:
        self.records: List[PageRecord] = []
        self.alive = np.zeros(0, dtype=bool)
        self._n = 0
        self._by_doc: Dict[str, List[int]] = {}
        self._by_key: Dict[Tuple[str, int], int] = {}
        # columnar copies of document_id / app_id as small integers: the doc_ids filter becomes one table gather
        self._doc_index: Dict[str, int] = {}
        self._app_index: Dict[str, int] = {}
        self._page_doc = np.zeros(0, dtype=np.int32)
        self._page_app = np.zeros(0, dtype=np.int32)  # -1 = stored without an app_id (visible to everybody)
        self.version = 0  # bumped by every mutation; keys the mask cache
        self._mask_cache: "OrderedDict[Tuple, Optional[np.ndarray]]" = OrderedDict()

    # ------------------------------------------------------------------ size
    def __len__(self) -> int:
        return self._n

    @property
    def n_live(self) -> int:
        return int(self.alive[: self._n].sum())

    @property
    def dead_fraction(self) -> float:
        return 0.0 if self._n == 0 else 1.0 - self.n_live / self._n

    # ------------------------------------------------------------------ writes
    def add(self, rec: PageRecord) -> int:
        pid = self._n
        if pid >= self.alive.shape[0]:
            cap = max(1024, 2 * self.alive.shape[0])
            for name, dt in (("alive", bool), ("_page_doc", np.int32), ("_page_app", np.int32)):
                grown = np.zeros(cap, dtype=dt)
                grown[: self._n] = getattr(self, name)[: self._n]
                setattr(self, name, grown)
        self.records.append(rec)
        self.alive[pid] = True
        self._page_doc[pid] = self._doc_index.setdefault(rec.document_id, len(self._doc_index))
        self._page_app[pid] = -1 if rec.app_id is None else self._app_index.setdefault(rec.app_id, len(self._app_index))
        self._n += 1
        self.version += 1
        self._by_doc.setdefault(rec.document_id, []).append(pid)
        self._by_key[(rec.document_id, int(rec.chunk_number))] = pid  # a re-insert of the same key shadows the old page
        return pid

    def delete_document(self, document_id: str) -> List[int]:
        pids = self._by_doc.pop(document_id, [])
        self.version += 1
        for pid in pids:
            self.alive[pid] = False
            rec = self.records[pid]
            if self._by_key.get((rec.document_id, int(rec.chunk_number))) == pid:
                del self._by_key[(rec.document_id, int(rec.chunk_number))]
        return pids

    # ------------------------------------------------------------------ reads
    def lookup(self, document_id: str, chunk_number: int) -> Optional[int]:
        pid = self._by_key.get((document_id, int(chunk_number)))
        return pid if pid is not None and self.alive[pid] else None

    @property
    def n_documents(self) -> int:
        """Number of document ordinals handed out (page_documents() values lie in [0, n_documents))."""
        return len(self._doc_index)

    def page_documents(self) -> np.ndarray:
        """int32 [n_pages]: the document ordinal of every page, -1 for a deleted page (the table the grouped search reads)."""
        n = self._n
        return np.where(self.alive[:n], self._page_doc[:n], -1).astype(np.int32)

    def pages_of(self, document_id: str) -> List[int]:
        return [p for p in self._by_doc.get(document_id, []) if self.alive[p]]

    def allow_mask(self, doc_ids: Optional[Sequence[str]] = None, app_id: Optional[str] = None) -> Optional[np.ndarray]:
        """bool[n_pages] of pages a query may return, or None when every page qualifies (no mask upload needed).

        doc_ids=None means "no document filter" (multi_vector_store.py:752); an EMPTY list selects nothing.
        A page stored with an app_id is only visible to queries with the same app_id (the fast store's namespace,
        fast_multivector_store.py:311,526); pages stored without one are visible to everybody.
        """
        n = self._n
        mask = self.alive[:n].copy()
        if doc_ids is not None:
            lut = np.zeros(len(self._doc_index) + 1, dtype=bool)
            idx = [self._doc_index[d] for d in doc_ids if d in self._doc_index]
            if idx:
                lut[idx] = True
            mask &= lut[self._page_doc[:n]]
        if app_id is not None:
            mine = self._app_index.get(app_id, -2)
            pa = self._page_app[:n]
            mask &= (pa < 0) | (pa == mine)
        return None if mask.all() else mask

    def allow_words(self, doc_ids: Optional[Sequence[str]] = None, app_id: Optional[str] = None
                    ) -> Tuple[bool, Optional[np.ndarray]]:
        """(any page visible?, device filter words or None = unfiltered) with a small LRU: a user's authorised document
        list (document_service.py:408-417) repeats from query to query, so the mask is usually a dictionary hit."""
        key = (self.version, app_id, None if doc_ids is None else tuple(doc_ids))
        hit = self._mask_cache.get(key, False)
        if hit is not False:
            self._mask_cache.move_to_end(key)
            return hit
        mask = self.allow_mask(doc_ids, app_id)
        val = (True, None) if mask is None else (bool(mask.any()), self.mask_words(mask))
        self._mask_cache[key] = val
        while len(self._mask_cache) > 64:
            self._mask_cache.popitem(last=False)
        return val

    @staticmethod
    def mask_words(mask: np.ndarray) -> np.ndarray:
        """bool[n] -> uint32 words, bit p&31 of word p>>5 (the device filter format of b200ms_topk)."""
        pad = (-len(mask)) % 32
        bits = np.concatenate([mask, np.zeros(pad, dtype=bool)]) if pad else mask
        if len(bits) == 0:
            return np.zeros(0, dtype=np.uint32)
        return np.packbits(bits.reshape(-1, 32), axis=1, bitorder="little").view(np.uint32).reshape(-1).copy()

    @staticmethod
    def stack_masks(masks: Sequence[Optional[np.ndarray]]) -> Tuple[Optional[np.ndarray], List[int]]:
        """One word array (or None = unfiltered) per query -> (matrix [n_distinct, words] with one row per distinct mask, or
        None when no query is filtered; each query's row, -1 = unfiltered): the per-query filter format of the library.
        Users sharing a filter share a row, so it is uploaded once."""
        rows, index, seen = [], [], {}
        for m in masks:
            if m is None:
                index.append(-1)
                continue
            key = m.tobytes()
            if key not in seen:
                seen[key] = len(rows)
                rows.append(m)
            index.append(seen[key])
        return (np.stack(rows) if rows else None), index

    # ------------------------------------------------------------------ compaction
    def compaction_plan(self) -> Tuple[np.ndarray, np.ndarray]:
        """(kept old page ids in order, old->new id map with -1 for dropped pages)."""
        keep = np.nonzero(self.alive[: self._n])[0]
        remap = np.full(self._n, -1, dtype=np.int64)
        remap[keep] = np.arange(len(keep))
        return keep, remap

    def apply_compaction(self, keep: Iterable[int]) -> None:
        old = self.records
        self.records, self._by_doc, self._by_key = [], {}, {}
        self._doc_index, self._app_index = {}, {}
        self.alive = np.zeros(0, dtype=bool)
        self._page_doc = np.zeros(0, dtype=np.int32)
        self._page_app = np.zeros(0, dtype=np.int32)
        self._mask_cache.clear()
        self._n = 0
        for pid in keep:
            self.add(old[int(pid)])
