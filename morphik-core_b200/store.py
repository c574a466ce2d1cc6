"""B200MultiVectorStore -- the drop-in ``BaseVectorStore`` for Morphik's ColPali (multi-vector) retrieval.

Keeps the plugin contract of core/vector_store/base_vector_store.py:7-65 byte for byte (four async methods, same
argument names/meaning, same return shapes) plus the de-facto extras callers use: ``initialize()``
(core/app_factory.py:78-80), ``close()``, and the ``.storage`` / ``.uri`` attributes
(core/vector_store/dual_multivector_store.py:224-232).  Semantics follow the two reference providers:

  provider "postgres" (MultiVectorStore, multi_vector_store.py)   -> ``mode="binary"``: sign-bit quantise, exhaustive
      Hamming MaxSim, score = SQL max_sim value (multiples of 1/128), ORDER BY score DESC LIMIT k.
  provider "morphik" (FastMultiVectorStore, fast_multivector_store.py) -> ``mode="bf16"``: float MaxSim; the reference
      reranks <=75 ANN candidates, this store scores EVERY authorised page exactly (a superset of that behaviour).
  ``mode="int8"`` is new (BASELINE config 3).

Everything heavy runs on the GPU through libb200ms (see index.py); this class only owns the id <-> (document, chunk)
catalogue, the doc_ids -> page-mask conversion, payload bookkeeping and DocumentChunk construction.  GPU calls are
serialised with a lock and pushed off the event loop with asyncio.to_thread (SURVEY 8b "Threading").

Concurrent ``query_similar`` coroutines (the API server's situation) are COALESCED: while one GPU pass is running, the
requests that arrive queue up and the next pass scores them together, each against its own authorised-page mask
(``b200ms_search_host_masked``).  A single 32-token query leaves 3/4 of every 128-row MMA tile empty and the scan is
HBM-bound, so up to ~8 queries ride for the price of one; a lone query is not delayed (there is no batching window).
"""
from __future__ import annotations

import asyncio
import collections
import dataclasses
import json
import logging
import threading
import time
import weakref
from typing import Any, Dict, List, Optional, Sequence, Tuple

import numpy as np

from .catalog import PageCatalog, PageRecord
from .models import DocumentChunk

logger = logging.getLogger(__name__)
MAX_K = 4096  # B200MS_MAX_K
# metadata key of the document score on the chunks query_similar_documents(score_by="document") returns
DOCUMENT_SCORE_KEY = "document_score"
# metadata key of the other visible members of a chunk's duplicate group on the chunks query_similar_distinct returns
DUPLICATES_KEY = "duplicates"

try:  # inside a Morphik checkout the reference ABC is the real base class
    from core.vector_store.base_vector_store import BaseVectorStore  # type: ignore
except Exception:  # standalone: same abstract surface
    from abc import ABC, abstractmethod

    class BaseVectorStore(ABC):  # mirrors core/vector_store/base_vector_store.py:7-65
        @abstractmethod
        async def store_embeddings(self, chunks, app_id=None): ...

        @abstractmethod
        async def query_similar(self, query_embedding, k, doc_ids=None, app_id=None, skip_image_content=False): ...

        @abstractmethod
        async def get_chunks_by_id(self, chunk_identifiers, app_id=None, skip_image_content=False): ...

        @abstractmethod
        async def delete_chunks_by_document_id(self, document_id, app_id=None): ...


def build_store_metrics(**kw) -> Dict[str, Any]:
    """Same keys as core/vector_store/utils.py:73-103 so ingestion telemetry keeps working."""
    base = dict(chunk_payload_upload_s=0.0, chunk_payload_objects=0, chunk_payload_bytes=0, chunk_payload_backend="memory",
                multivector_upload_s=0.0, multivector_objects=0, multivector_bytes=0, multivector_backend="b200-hbm",
                vector_store_write_s=0.0, vector_store_backend="b200-hbm", vector_store_rows=0, cache_write_s=0.0,
                cache_write_objects=0)
    base.update(kw)
    return base


def _document_chunk(rec: PageRecord, score) -> DocumentChunk:
    """The DocumentChunk a search returns for a stored page (its embedding is not sent back)."""
    return DocumentChunk(document_id=rec.document_id, chunk_number=rec.chunk_number, content=rec.content, embedding=[],
                         metadata=dict(rec.metadata), score=float(score))


def _capped_k(k: int) -> int:
    """k limited to what one top-k call returns (B200MS_MAX_K), with a warning when that truncates it."""
    if k > MAX_K:
        logger.warning("k=%d requested; truncated to %d (B200MS_MAX_K)", k, MAX_K)
    return min(int(k), MAX_K)


def as_query_matrix(query_embedding) -> np.ndarray:
    """np.ndarray | torch.Tensor | List[np.ndarray] | List[torch.Tensor] | nested lists -> float32 [T,128]
    (accepted input forms: multi_vector_store.py:723,334-337; fast_multivector_store.py:506,515-518)."""
    try:
        import torch

        if isinstance(query_embedding, torch.Tensor):
            query_embedding = query_embedding.detach().float().cpu().numpy()
        elif isinstance(query_embedding, (list, tuple)) and len(query_embedding) and isinstance(query_embedding[0], torch.Tensor):
            query_embedding = np.stack([t.detach().float().cpu().numpy() for t in query_embedding])
    except ImportError:  # pragma: no cover
        pass
    q = np.asarray(query_embedding, dtype=np.float32)
    if q.ndim == 1:
        q = q[None, :]
    if q.ndim != 2 or q.shape[1] != 128:
        raise ValueError(f"query embedding must be [T,128], got {q.shape}")
    return np.ascontiguousarray(q)


def as_page_matrix(embedding):
    """Page embedding -> [P,128] matrix for ``add_pages``.

    CUDA torch tensors (what ColpaliEmbeddingModel holds before its ``.to(float32).numpy(force=True)``,
    colpali_embedding_model.py:262,291) stay on the device as bf16/float32 and go straight into the pack kernel -- the
    ingest fast path (SURVEY 8f-3): no fp32 host copy, no Rust pack, no ``Bit`` objects, no ``executemany``
    (multi_vector_store.py:681-703).  Everything else becomes a host float32 array, as the reference does (:334-337)."""
    if hasattr(embedding, "detach"):
        t = embedding.detach()
        if t.is_cuda:
            import torch

            if t.dtype not in (torch.bfloat16, torch.float32):
                t = t.float()
            return t[None, :] if t.ndim == 1 else t
        embedding = t.float().cpu().numpy()
    emb = np.asarray(embedding, dtype=np.float32)
    return emb[None, :] if emb.ndim == 1 else emb


class _QueryRequest:
    __slots__ = ("q", "k", "doc_ids", "app_id", "future")

    def __init__(self, q, k, doc_ids, app_id, future):
        self.q, self.k, self.doc_ids, self.app_id, self.future = q, k, doc_ids, app_id, future


class _LoopQueue:
    """Pending query_similar requests of ONE event loop and the task that drains them."""
    __slots__ = ("pending", "task", "__weakref__")

    def __init__(self):
        self.pending = collections.deque()
        self.task = None


class QueryCoalescer:
    """Mixin: concurrent ``query_similar`` coroutines share GPU passes.  The host class provides
    ``_search_coalesced_locked(batch) -> List[List[DocumentChunk]]`` (runs in a worker thread) and calls
    ``_init_coalescer`` in its constructor."""

    def _init_coalescer(self, coalesce_queries: bool, max_coalesced_tokens: int, max_coalesced_queries: int) -> None:
        # 1024 tokens = one CTA-pair pass over the corpus
        self.coalesce_queries = bool(coalesce_queries)
        self.max_coalesced_tokens = int(max_coalesced_tokens)
        self.max_coalesced_queries = int(max_coalesced_queries)
        self._queues: "weakref.WeakKeyDictionary[Any, _LoopQueue]" = weakref.WeakKeyDictionary()
        self._queues_lock = threading.Lock()
        self.last_coalesced_batch = 0

    async def _enqueue_query(self, q: np.ndarray, k: int, doc_ids, app_id) -> List[DocumentChunk]:
        loop = asyncio.get_running_loop()
        with self._queues_lock:
            lq = self._queues.get(loop)
            if lq is None:
                lq = self._queues[loop] = _LoopQueue()
        req = _QueryRequest(q, int(k), doc_ids, app_id, loop.create_future())
        lq.pending.append(req)
        if lq.task is None or lq.task.done():
            lq.task = loop.create_task(self._drain(lq))
        return await req.future

    async def _drain(self, lq: _LoopQueue) -> None:
        """Score everything that is pending, one GPU pass per batch; requests arriving meanwhile form the next batch."""
        while lq.pending:
            batch, tokens = [], 0
            while lq.pending and len(batch) < self.max_coalesced_queries:
                nxt = lq.pending[0]
                if batch and tokens + nxt.q.shape[0] > self.max_coalesced_tokens:
                    break
                batch.append(lq.pending.popleft())
                tokens += nxt.q.shape[0]
            try:
                results = await asyncio.to_thread(self._search_coalesced_locked, batch)
            except BaseException as e:  # noqa: BLE001  (every waiter must be released; errors propagate like the reference's)
                for r in batch:
                    if not r.future.done():
                        r.future.set_exception(e if isinstance(e, Exception) else RuntimeError(repr(e)))
                if not isinstance(e, Exception):
                    raise
                continue
            self.last_coalesced_batch = len(batch)
            for r, res in zip(batch, results):
                if not r.future.done():
                    r.future.set_result(res)


class B200MultiVectorStore(QueryCoalescer, BaseVectorStore):
    """Exhaustive ColPali MaxSim store on one H100 (see module docstring)."""

    def __init__(self, uri: str = "b200://0", device: int = 0, mode: str = "bf16", storage: Any = None,
                 auto_initialize: bool = True, compact_dead_fraction: float = 0.3, index: Any = None,
                 fde_candidates: Optional[int] = None, coalesce_queries: bool = True, max_coalesced_tokens: int = 1024,
                 max_coalesced_queries: int = 64, zero_pad_compat: int = 0, corpus_tier: str = "hbm",
                 sign_candidates: Optional[int] = None):
        # corpus_tier "host": patch rows in pinned host memory, bounded by host RAM instead of HBM; only the candidates of a
        # query cross PCIe (the reference's load_multivector_from_storage, fast_multivector_store.py:545-548), so it needs
        # the two-stage search
        if corpus_tier not in ("hbm", "host"):
            raise ValueError(f"corpus_tier must be 'hbm' or 'host', got {corpus_tier!r}")
        if fde_candidates and sign_candidates:
            raise ValueError("fde_candidates and sign_candidates are two first stages of the two-stage search: pass one")
        if corpus_tier == "host" and not (fde_candidates or sign_candidates):
            raise ValueError("corpus_tier='host' needs fde_candidates or sign_candidates: a host-resident corpus is only scored "
                             "on candidate lists")
        self.corpus_tier = corpus_tier
        self.uri = uri
        self.device = int(device)
        self.mode = mode
        self.storage = storage  # attribute kept for DualMultiVectorStore / DocumentService compatibility
        # Tombstoned pages cost HBM until the compaction, but no scan time once any filter is given: the catalogue's masks
        # clear them (PageCatalog.allow_mask starts from `alive`), and a filtered search reads only the pages its mask allows.
        self.compact_dead_fraction = float(compact_dead_fraction)
        self.catalog = PageCatalog()
        self._index = index  # injectable for host-logic tests; the product builds a MaxSimIndex in initialize()
        # None: exhaustive MaxSim over every authorised page (Postgres-provider behaviour).  An int: two-stage search like
        # the "morphik" provider -- FDE candidates (the reference asks Turbopuffer for min(10*k, 75)) then MaxSim rerank.
        self.fde_candidates = fde_candidates
        # An int: the same two-stage search with the asymmetric sign scan as its first stage (signs.SignTwoStageIndex:
        # full-precision queries against an HBM sign copy of every page) instead of the FDE scan.
        self.sign_candidates = sign_candidates
        self._n_candidates = int(fde_candidates or sign_candidates or 0)
        self._two_stage = None  # the first stage with the rerank behind it (two_stage.TwoStageSearch) in two-stage mode
        # > 0: reproduce colpali_engine score_multi_vector's zero-padding quirk with this batch size (128 upstream): a page
        # shorter than the longest page of its scoring batch scores sum_t max(max_r <q_t,d_r>, 0)  (SURVEY App. A.2;
        # processing_colpali.py:350-362).  0 (default) = the clean MaxSim.
        self.zero_pad_compat = int(zero_pad_compat)
        self._init_coalescer(coalesce_queries, max_coalesced_tokens, max_coalesced_queries)  # see module docstring
        self._lock = threading.Lock()
        self._journal = None  # shardfile.StoreJournal when the store is durable (B200MultiVectorStore.open)
        self._last_store_metrics: Dict[str, Any] = {}
        self.last_query_timing: Dict[str, float] = {}
        self._page_doc_cache: Optional[Tuple[int, Any]] = None  # (catalog.version, device page -> document table)
        # index_duplicates' pair table (device pair_a, pair_b, sim_ab, sim_ba) and the pages it has taken as sources;
        # None until the first call, not persisted
        self._dup: Optional[Dict[str, Any]] = None
        if auto_initialize:
            self.initialize()

    # ------------------------------------------------------------------ lifecycle
    def initialize(self) -> bool:
        if self._index is None:
            from .index import MaxSimIndex  # raises when libb200ms.so or the GPU is missing: no silent fallback

            if self._n_candidates:
                self._two_stage = self._first_stage(index=None, device=self.device, dtype=self.mode, tier=self.corpus_tier)
                self._index = self._two_stage.index
            else:
                self._index = MaxSimIndex(device=self.device, dtype=self.mode)
        elif self._n_candidates and self._two_stage is None and hasattr(self._index, "h"):
            # a loaded / injected CUDA index in two-stage mode: rebuild the first stage's rows from its packed rows
            self._two_stage = self._first_stage(index=self._index)
            self._two_stage.rebuild_from_index()
        if self.zero_pad_compat and hasattr(self._index, "set_option"):
            self._index.set_option("zero_pad_compat", self.zero_pad_compat)
        return True

    def _first_stage(self, **kw):
        from .fde import TwoStageIndex
        from .signs import SignTwoStageIndex

        return (TwoStageIndex if self.fde_candidates else SignTwoStageIndex)(**kw)

    def close(self) -> None:
        if self._index is not None and hasattr(self._index, "close"):
            self._index.close()
        self._index = None

    def latest_store_metrics(self) -> Dict[str, Any]:
        return dict(self._last_store_metrics)

    # ------------------------------------------------------------------ write path
    async def store_embeddings(self, chunks: List[DocumentChunk], app_id: Optional[str] = None
                               ) -> Tuple[bool, List[str], Dict[str, Any]]:
        valid = []
        for c in chunks:
            if getattr(c, "embedding", None) is None:
                logger.error("Missing embeddings for chunk %s-%s", c.document_id, c.chunk_number)
                continue
            emb = as_page_matrix(c.embedding)
            if emb.ndim != 2 or emb.shape[1] != 128:
                raise ValueError(f"chunk {c.document_id}-{c.chunk_number}: embedding must be [P,128], got {tuple(emb.shape)}")
            valid.append((c, emb))
        if not valid:
            self._last_store_metrics = build_store_metrics()
            return True, [], self._last_store_metrics
        t0 = time.perf_counter()
        await asyncio.to_thread(self._add_pages_locked, valid, app_id)
        dt = time.perf_counter() - t0
        self._last_store_metrics = build_store_metrics(
            vector_store_write_s=dt, vector_store_rows=len(valid), multivector_objects=len(valid), multivector_upload_s=dt,
            multivector_bytes=int(sum(e.shape[0] for _, e in valid)) * self._index.row_bytes)
        return True, [f"{c.document_id}-{c.chunk_number}" for c, _ in valid], self._last_store_metrics

    def _add_pages_locked(self, valid, app_id):
        with self._lock:
            first, n = (self._two_stage or self._index).add_pages([e for _, e in valid])
            recs = []
            for i, (c, e) in enumerate(valid):
                rec = PageRecord(c.document_id, int(c.chunk_number), c.content, dict(c.metadata or {}), app_id, int(e.shape[0]))
                pid = self.catalog.add(rec)
                assert pid == first + i, "catalogue and device corpus out of step"
                recs.append(rec)
            if self._journal is not None:  # durable store: this call becomes one append-only segment
                self._journal.log_add(self._index, first, n, [dataclasses.asdict(r) for r in recs], self._journal_rows(first, n))

    def _journal_rows(self, first: int, n: int):
        """What a journal segment persists of the first stage (FDE rows; sign rows are derived again on replay)."""
        return self._two_stage.journal_rows(first, n) if self._two_stage is not None else None

    # ------------------------------------------------------------------ read path
    async def query_similar(self, query_embedding, k: int, doc_ids: Optional[List[str]] = None,
                            app_id: Optional[str] = None, skip_image_content: bool = False) -> List[DocumentChunk]:
        if not self.coalesce_queries:
            results = await self.query_similar_batch([query_embedding], k, doc_ids, app_id, skip_image_content)
            return results[0]
        q = as_query_matrix(query_embedding)
        if k <= 0:
            return []
        return await self._enqueue_query(q, k, doc_ids, app_id)

    def _search_coalesced_locked(self, batch: List[_QueryRequest]) -> List[List[DocumentChunk]]:
        """One pass for a batch of independent requests; masks are built under the lock so they match the corpus."""
        t0 = time.perf_counter()
        with self._lock:
            n = len(self.catalog)
            out: List[Optional[List[DocumentChunk]]] = [None] * len(batch)
            live = []
            for i, r in enumerate(batch):
                visible, words = self.catalog.allow_words(r.doc_ids, r.app_id) if n else (False, None)
                if not visible:
                    out[i] = []
                else:
                    live.append((i, r, words))
            if live:
                kk = min(_capped_k(max(r.k for _, r, _ in live)), n)
                queries = [r.q for _, r, _ in live]
                masks = [w for _, _, w in live]
                if self._two_stage is None and hasattr(self._index, "search_host_masked") and len(live) > 1:
                    ts, ti, tc = self._index.search_host_masked(queries, kk, masks)
                else:  # two-stage search / injected test index: one call per distinct mask
                    ts = np.full((len(live), kk), -np.inf, dtype=np.float32)
                    ti = np.full((len(live), kk), -1, dtype=np.int64)
                    tc = np.zeros((len(live),), dtype=np.int32)
                    groups: Dict[Optional[bytes], List[int]] = {}
                    for j, w in enumerate(masks):
                        groups.setdefault(None if w is None else w.tobytes(), []).append(j)
                    for idxs in groups.values():
                        a, b, c = self._search_unlocked([queries[j] for j in idxs], kk, masks[idxs[0]])
                        ts[idxs], ti[idxs], tc[idxs] = a, b, c
                for row, (i, r, _) in enumerate(live):
                    out[i] = self._chunks(ts[row], ti[row], min(int(tc[row]), r.k))
        self.last_query_timing = {"coalesced_queries": float(len(batch)), "total_ms": (time.perf_counter() - t0) * 1e3}
        return out  # type: ignore[return-value]

    def _chunks(self, scores, ids, count: int, min_score: Optional[float] = None) -> List[DocumentChunk]:
        hits = []
        for j in range(count):
            if min_score is not None and float(scores[j]) < min_score:
                break  # sorted by score descending
            hits.append(_document_chunk(self.catalog.records[int(ids[j])], scores[j]))
        return hits

    async def query_similar_batch(self, query_embeddings: Sequence[Any], k: int, doc_ids: Optional[List[str]] = None,
                                  app_id: Optional[str] = None, skip_image_content: bool = False,
                                  min_score: Optional[float] = None) -> List[List[DocumentChunk]]:
        """Batched form (extension): one corpus pass scores every query of the batch.

        ``min_score`` drops hits scoring below it (the reference accepts ``min_score`` in retrieve_chunks but never applies
        it, document_service.py:381-383; SURVEY 8f-4) -- scores are MaxSim sums, so the threshold is on that scale.
        Mask construction, the GPU search and the id -> DocumentChunk resolution run in ONE worker-thread call under the
        store lock, so an ingest or compaction can never slip between them."""
        queries = [as_query_matrix(q) for q in query_embeddings]
        if k <= 0:
            return [[] for _ in queries]
        return await asyncio.to_thread(self._search_batch_locked, queries, int(k), doc_ids, app_id, min_score)

    def _search_batch_locked(self, queries, k, doc_ids, app_id, min_score):
        t0 = time.perf_counter()
        with self._lock:
            n = len(self.catalog)
            if n == 0:
                return [[] for _ in queries]
            visible, words = self.catalog.allow_words(doc_ids, app_id)
            if not visible:
                return [[] for _ in queries]
            kk = min(_capped_k(k), n)
            t1 = time.perf_counter()
            ts, ti, tc = self._search_unlocked(queries, kk, words)
            t2 = time.perf_counter()
            out = [self._chunks(ts[qi], ti[qi], int(tc[qi]), min_score) for qi in range(len(queries))]
            t3 = time.perf_counter()
        self.last_query_timing = {"prepare_ms": (t1 - t0) * 1e3, "gpu_search_ms": (t2 - t1) * 1e3,
                                  "build_chunks_ms": (t3 - t2) * 1e3, "total_ms": (t3 - t0) * 1e3}
        if self._two_stage is not None:  # the reference's stage names (fast_multivector_store.py:523,534,550,574,589,604)
            self.last_query_timing.update({k: float(v) for k, v in self._two_stage.last_timing_ms.items()},
                                          load_contents_ms=0.0)
        logger.debug("query_similar timing %s", json.dumps(self.last_query_timing))
        return out

    def _search_locked(self, queries, k, words):
        with self._lock:
            return self._search_unlocked(queries, k, words)

    def _search_unlocked(self, queries, k, words):
        if self._two_stage is not None:
            return self._two_stage.search(queries, k, n_candidates=max(self._n_candidates, k), allow_mask=words)
        return self._index.search_host(queries, k, allow_mask=words)

    async def query_similar_documents(self, query_embedding, k: int, pages_per_document: int = 1,
                                      doc_ids: Optional[List[str]] = None, app_id: Optional[str] = None,
                                      min_score: Optional[float] = None, score_by: str = "page") -> List[List[DocumentChunk]]:
        """The top k DOCUMENTS instead of the top k chunks (extension): one list per document, best document first.

        ``score_by="page"`` (default): a document ranks by its best chunk, and each list holds that document's best
        ``pages_per_document`` chunks in score order with query_similar's scores -- query_similar's ranking grouped by
        document, computed on the GPU without over-fetching chunks.  ``min_score`` drops chunks below it and a document
        left without chunks.

        ``score_by="document"``: a document is scored as one bag of patches, each query token taking its best patch on ANY
        of the document's pages (document-level MaxSim), so a document that answers different parts of the query on
        different pages ranks as one match.  Longer documents are favoured: the score only grows with pages, and nothing
        normalises it.  Each list holds the document's evidence chunks -- the pages holding some token's best patch, at most
        ``pages_per_document``, largest share first -- and a chunk's ``score`` is its share (the token maxima it holds);
        the document's score is in every chunk's ``metadata["document_score"]``.  ``min_score`` drops documents whose
        score is below it.  Needs an HBM-tier index.

        ``doc_ids`` / ``app_id`` filter as in query_similar.  Mask, GPU search and chunk construction are one critical
        section."""
        q = as_query_matrix(query_embedding)
        per = int(pages_per_document)
        if not 1 <= per <= 64:
            raise ValueError("pages_per_document must be in [1, 64]")
        if score_by not in ("page", "document"):
            raise ValueError(f"score_by must be 'page' or 'document', got {score_by!r}")
        if k <= 0:
            return []
        return await asyncio.to_thread(self._search_docs_locked, q, int(k), per, doc_ids, app_id, min_score, score_by)

    def _page_doc_table(self):
        import torch

        if self._page_doc_cache is None or self._page_doc_cache[0] != self.catalog.version:
            table = torch.from_numpy(self.catalog.page_documents()).to(self._index.device)
            self._page_doc_cache = (self.catalog.version, table)
        return self._page_doc_cache[1]

    def _search_docs_locked(self, q, k, per, doc_ids, app_id, min_score, score_by="page"):
        with self._lock:
            n = len(self.catalog)
            if n == 0:
                return []
            visible, words = self.catalog.allow_words(doc_ids, app_id)
            if not visible:
                return []
            n_docs = self.catalog.n_documents
            kk = min(_capped_k(k), n_docs)
            page_doc = self._page_doc_table()
            if score_by == "document":
                return self._doc_maxsim_unlocked(q, kk, per, page_doc, n_docs, words, min_score)
            if self._two_stage is not None:
                ts, ti, pc, dc = self._two_stage.search_docs([q], kk, per, page_doc, n_docs,
                                                             n_candidates=max(self._n_candidates, kk * per), allow_mask=words)
            else:
                ts, ti, pc, dc = self._index.search_docs([q], kk, per, page_doc, n_docs, allow_mask=words)
            out = []
            for i in range(int(dc[0])):
                chunks = self._chunks(ts[0, i], ti[0, i], int(pc[0, i]), min_score)
                if chunks:
                    out.append(chunks)
            return out

    def _doc_maxsim_unlocked(self, q, k, per, page_doc, n_docs, words, min_score):
        if self._two_stage is not None:
            ds, di, ei, es, ec, dc = self._two_stage.search_doc_maxsim([q], k, per, page_doc, n_docs,
                                                                       n_candidates=max(self._n_candidates, k), allow_mask=words)
        else:
            ds, di, ei, es, ec, dc = self._index.search_doc_maxsim([q], k, per, page_doc, n_docs, allow_mask=words)
        out = []
        for i in range(int(dc[0])):
            score = float(ds[0, i])
            if min_score is not None and score < min_score:
                break  # sorted by document score descending
            chunks = self._chunks(es[0, i], ei[0, i], int(ec[0, i]))
            for c in chunks:
                c.metadata[DOCUMENT_SCORE_KEY] = score
            out.append(chunks)
        return out

    async def query_similar_mmr(self, query_embedding, k: int, fetch_k: int = 20, lambda_mult: float = 0.5,
                                doc_ids: Optional[List[str]] = None, app_id: Optional[str] = None) -> List[DocumentChunk]:
        """k chunks that are relevant AND different from each other (extension; LangChain's
        ``max_marginal_relevance_search``): the store's own search (exhaustive or two-stage) fetches the best
        ``max(fetch_k, k)`` chunks under the ``doc_ids`` / ``app_id`` filter, then maximal marginal relevance picks k of them on
        the GPU (MaxSimIndex.mmr): first the best chunk, then each time the chunk maximising ``lambda_mult`` * relevance -
        (1 - ``lambda_mult``) * its page-to-page MaxSim against the chunks picked already.  ``lambda_mult`` = 1 is
        query_similar's ranking, 0 the most diverse.  Chunks come in pick order with query_similar's scores.  Mask, search,
        MMR and chunk construction are one critical section; ``last_query_timing["mmr_ms"]`` is the MMR call's device time."""
        q = as_query_matrix(query_embedding)
        if not 0.0 <= float(lambda_mult) <= 1.0:  # NaN fails too
            raise ValueError(f"lambda_mult must be in [0, 1], got {lambda_mult}")
        if k <= 0:
            return []
        return await asyncio.to_thread(self._search_mmr_locked, q, int(k), int(fetch_k), float(lambda_mult), doc_ids, app_id)

    def _search_mmr_locked(self, q, k, fetch_k, lambda_mult, doc_ids, app_id):
        import torch

        t0 = time.perf_counter()
        with self._lock:
            n = len(self.catalog)
            if n == 0:
                return []
            visible, words = self.catalog.allow_words(doc_ids, app_id)
            if not visible:
                return []
            fetch = min(_capped_k(max(fetch_k, k)), n)
            t1 = time.perf_counter()
            ts, ti, tc = self._search_unlocked([q], fetch, words)
            t2 = time.perf_counter()
            count = int(tc[0])
            if count == 0:
                return []
            dev = torch.device(self._index.device)
            cand_ids = torch.from_numpy(np.ascontiguousarray(ti[:1, :count], dtype=np.int64)).to(dev)
            cand_scores = torch.from_numpy(np.ascontiguousarray(ts[:1, :count], dtype=np.float32)).to(dev)
            ev = [torch.cuda.Event(enable_timing=True) for _ in range(2)] if dev.type == "cuda" else None
            if ev:
                ev[0].record(torch.cuda.current_stream(dev))
            mi, ms, mc = self._index.mmr(cand_ids, cand_scores, [int(q.shape[0])], min(k, count), lambda_mult)
            if ev:
                ev[1].record(torch.cuda.current_stream(dev))
            mi, ms, mc = (np.asarray(t.cpu()) for t in (mi, ms, mc))  # waits for the call
            t3 = time.perf_counter()
            mmr_ms = ev[0].elapsed_time(ev[1]) if ev else (t3 - t2) * 1e3
            out = self._chunks(ms[0], mi[0], int(mc[0]))
            t4 = time.perf_counter()
        self.last_query_timing = {"prepare_ms": (t1 - t0) * 1e3, "gpu_search_ms": (t2 - t1) * 1e3, "mmr_ms": float(mmr_ms),
                                  "build_chunks_ms": (t4 - t3) * 1e3, "total_ms": (t4 - t0) * 1e3}
        if self._two_stage is not None:
            self.last_query_timing.update({k: float(v) for k, v in self._two_stage.last_timing_ms.items()})
        return out

    # ------------------------------------------------------------------ near-duplicate pages
    def _refuse_duplicates_on_host_tier(self):
        if self.corpus_tier != "hbm":
            raise ValueError("duplicate detection needs an HBM-tier store (corpus_tier='hbm'): the pair kernel reads both "
                             "pages of a pair from HBM")

    async def index_duplicates(self, n_candidates: int = 10, rebuild: bool = False) -> int:
        """Build or extend the near-duplicate pair table (extension; a maintenance call, like compaction): every live page
        added since the previous call is a source, its ``n_candidates`` most similar live pages (the store's first stage
        in two-stage mode, else search_pages) become candidate pairs, and one tensor-core product per pair scores both
        directions of page-to-page MaxSim (MaxSimIndex.pair_maxsim).  ``rebuild=True`` starts over with every live page as
        a source.  The table stays on the device; deletions drop out through the masks, compaction remaps it, and it is not
        persisted: after ``load`` / ``open`` call this again.  It holds the store lock for the whole build, as compaction
        does, so searches and ingests wait until it returns (seconds for tens of thousands of new pages; schedule it off
        peak).  Returns the number of pairs in the table.  HBM-tier stores only."""
        self._refuse_duplicates_on_host_tier()
        n_cand = int(n_candidates)
        if n_cand < 1:
            raise ValueError(f"n_candidates must be >= 1, got {n_candidates}")
        return await asyncio.to_thread(self._index_duplicates_locked, n_cand, bool(rebuild))

    def _index_duplicates_locked(self, n_cand, rebuild):
        import torch

        with self._lock:
            n = len(self.catalog)
            dev = torch.device(self._index.device)
            empty = torch.zeros((0,), dtype=torch.int64, device=dev)
            old = self._dup if (self._dup is not None and not rebuild) else {
                "a": empty, "b": empty, "sab": empty.float(), "sba": empty.float(), "n_indexed": 0}
            src = [p for p in range(old["n_indexed"], n) if self.catalog.alive[p]]
            a, b = empty, empty
            if src:
                _, words = self.catalog.allow_words(None, None)
                mask = None if words is None else torch.from_numpy(words.view(np.int32)).to(dev)
                target = self._two_stage if self._two_stage is not None else self._index
                a, b = target.duplicate_candidates(src, n_cand, mask)
            if a.numel():
                sab, sba = self._index.pair_maxsim(a, b)
                # the new pairs all have a page the old table never saw: concatenate and keep the table ordered by (a, b)
                a, b = torch.cat([old["a"], a]), torch.cat([old["b"], b])
                sab, sba = torch.cat([old["sab"], sab]), torch.cat([old["sba"], sba])
                order = torch.argsort(a * max(n, 1) + b)
                old = {"a": a[order].contiguous(), "b": b[order].contiguous(), "sab": sab[order].contiguous(),
                       "sba": sba[order].contiguous()}
            self._dup = dict(old, n_indexed=n)
            if dev.type == "cuda":
                torch.cuda.synchronize(dev)
            return int(self._dup["a"].numel())

    @staticmethod
    def _check_threshold(threshold) -> float:
        t = float(threshold)
        if not np.isfinite(t):
            raise ValueError(f"threshold must be a finite number, got {threshold}")
        return t

    def _duplicate_labels(self, threshold, words):
        """Duplicate labels of the visible pages (device int64 [n_pages], -1 for a page the request may not see): the
        cached pairs with both pages visible and min(sim_ab, sim_ba) >= threshold, joined into groups on the GPU.  Nothing is
        re-scored, and no group is joined through a page the request may not see."""
        import torch

        if self._dup is None:
            raise RuntimeError("no duplicate table: call index_duplicates() first (it is not persisted across load / open)")
        d = self._dup
        mask = None if words is None else torch.from_numpy(words.view(np.int32)).to(torch.device(self._index.device))
        return self._index.duplicate_groups(d["a"], d["b"], d["sab"], d["sba"], threshold, mask)

    async def find_duplicate_chunks(self, threshold: float, doc_ids: Optional[List[str]] = None,
                                    app_id: Optional[str] = None) -> List[List[DocumentChunk]]:
        """Groups of near-duplicate chunks (extension): pages joined by pairs of the index_duplicates table whose smaller
        direction of page-to-page MaxSim (per row, on the scale of query_similar_to_chunks' scores) reaches ``threshold``,
        among the chunks the ``doc_ids`` / ``app_id`` filter lets the caller see.  Returns every group of two or more chunks,
        groups by their first page and chunks in page order (score 0).  No threshold has been measured on real ColPali
        pages, so there is no default.  Needs index_duplicates() first; HBM-tier stores only."""
        self._refuse_duplicates_on_host_tier()
        t = self._check_threshold(threshold)
        return await asyncio.to_thread(self._find_duplicates_locked, t, doc_ids, app_id)

    def _find_duplicates_locked(self, threshold, doc_ids, app_id):
        with self._lock:
            if self._dup is None:
                raise RuntimeError("no duplicate table: call index_duplicates() first (it is not persisted across load / "
                                   "open)")
            n = len(self.catalog)
            if n == 0:
                return []
            visible, words = self.catalog.allow_words(doc_ids, app_id)
            if not visible:
                return []
            labels = self._duplicate_labels(threshold, words).cpu().numpy()
            pages = np.flatnonzero(labels >= 0)
            groups: Dict[int, List[int]] = {}
            for p in pages.tolist():
                groups.setdefault(int(labels[p]), []).append(p)
            return [[_document_chunk(self.catalog.records[p], 0.0) for p in g] for _, g in sorted(groups.items())
                    if len(g) > 1]

    async def query_similar_distinct(self, query_embedding, k: int, threshold: float, doc_ids: Optional[List[str]] = None,
                                     app_id: Optional[str] = None,
                                     min_score: Optional[float] = None) -> List[DocumentChunk]:
        """query_similar with near-duplicates collapsed (extension): the best chunk of each duplicate group
        (find_duplicate_chunks' groups at ``threshold``, among the chunks the filter lets the caller see), in query_similar's
        order and with its scores, k groups at most.  It is the store's grouped search (exhaustive or two-stage) with the
        duplicate labels as the page-to-group table.  Each chunk's ``metadata["duplicates"]`` lists the (document_id,
        chunk_number) of the other visible members of its group.  ``min_score`` drops chunks below it.  The labels are
        computed per request from the cached pairs (no page is re-scored).  No threshold has been measured on real ColPali
        pages, so there is no default.  Needs index_duplicates() first; HBM-tier stores only."""
        self._refuse_duplicates_on_host_tier()
        q = as_query_matrix(query_embedding)
        t = self._check_threshold(threshold)
        if self._dup is None:
            raise RuntimeError("no duplicate table: call index_duplicates() first (it is not persisted across load / open)")
        if k <= 0:
            return []
        return await asyncio.to_thread(self._search_distinct_locked, q, int(k), t, doc_ids, app_id, min_score)

    def _search_distinct_locked(self, q, k, threshold, doc_ids, app_id, min_score):
        import torch

        t0 = time.perf_counter()
        with self._lock:
            n = len(self.catalog)
            if n == 0:
                return []
            visible, words = self.catalog.allow_words(doc_ids, app_id)
            if not visible:
                return []
            kk = min(_capped_k(k), n)
            labels = self._duplicate_labels(threshold, words)
            t1 = time.perf_counter()
            group = labels.to(torch.int32).contiguous()  # -1: not visible, as a deleted page in the grouped search
            if self._two_stage is not None:
                ts, ti, pc, dc = self._two_stage.search_docs([q], kk, 1, group, n, n_candidates=max(self._n_candidates, kk),
                                                             allow_mask=words)
            else:
                ts, ti, pc, dc = self._index.search_docs([q], kk, 1, group, n, allow_mask=words)
            t2 = time.perf_counter()
            lab = labels.cpu().numpy()
            # the pages of each group as one slice of the pages sorted by label (one sort per request, not a scan per hit)
            by_label = np.argsort(lab, kind="stable")
            sorted_lab = lab[by_label]
            out = []
            for i in range(int(dc[0])):
                if int(pc[0, i]) < 1:
                    continue
                if min_score is not None and float(ts[0, i, 0]) < min_score:
                    break  # sorted by score descending
                p = int(ti[0, i, 0])
                chunk = _document_chunk(self.catalog.records[p], ts[0, i, 0])
                lo, hi = np.searchsorted(sorted_lab, lab[p], "left"), np.searchsorted(sorted_lab, lab[p], "right")
                chunk.metadata[DUPLICATES_KEY] = [(self.catalog.records[o].document_id, self.catalog.records[o].chunk_number)
                                                  for o in by_label[lo:hi].tolist() if o != p]
                out.append(chunk)
            t3 = time.perf_counter()
        self.last_query_timing = {"labels_ms": (t1 - t0) * 1e3, "gpu_search_ms": (t2 - t1) * 1e3,
                                  "build_chunks_ms": (t3 - t2) * 1e3, "total_ms": (t3 - t0) * 1e3}
        return out

    async def query_similar_to_chunks(self, chunk_identifiers: List[Tuple[str, int]], k: int,
                                      doc_ids: Optional[List[str]] = None, app_id: Optional[str] = None,
                                      include_same_document: bool = False,
                                      min_score: Optional[float] = None) -> List[List[DocumentChunk]]:
        """Chunks like stored chunks (extension; "query by id"): each named chunk's stored embedding is the query, as
        ``retrieve_chunks(query_image=...)`` would send a page-length query, without fetching or re-sending the embedding.
        One list per visible source chunk, in first-mention order, under the rules of ``get_chunks_by_id`` (unknown or
        deleted chunks and chunks of another ``app_id`` are skipped, duplicates collapsed).  ``doc_ids`` / ``app_id`` filter
        the results as in query_similar; the source chunk is never returned, and its document's other chunks only with
        ``include_same_document``.  Scores are page-to-page MaxSim per source row (query_similar's score for the source's
        rows over their count), so they compare across sources; ``min_score`` drops hits below it.  Every source of a call
        shares one pass over the corpus; masks, GPU search and chunk construction are one critical section."""
        if k <= 0 or not chunk_identifiers:
            return []
        return await asyncio.to_thread(self._similar_to_chunks_locked, list(chunk_identifiers), int(k), doc_ids, app_id,
                                       bool(include_same_document), min_score)

    def _similar_to_chunks_locked(self, chunk_identifiers, k, doc_ids, app_id, include_same_document, min_score):
        import torch

        t0 = time.perf_counter()
        with self._lock:
            recs = self._visible_records(chunk_identifiers, app_id)
            if not recs:
                return []
            n = len(self.catalog)
            base = self.catalog.allow_mask(doc_ids, app_id)
            base = self.catalog.alive[:n].copy() if base is None else base
            masks = []
            for pid, rec in recs:  # one row per source: the filter, minus the source (and, by default, its document)
                m = base.copy()
                m[pid] = False
                if not include_same_document:
                    m[self.catalog.pages_of(rec.document_id)] = False
                masks.append(m)
            if not any(m.any() for m in masks):
                return [[] for _ in recs]
            words = np.stack([PageCatalog.mask_words(m) for m in masks])
            kk = min(_capped_k(k), n)
            pids = [pid for pid, _ in recs]
            t1 = time.perf_counter()
            if self._two_stage is not None:  # each source's row filters its candidates too: no slot goes to an excluded page
                ts, ti, tc = self._two_stage.search_pages(pids, kk, n_candidates=max(self._n_candidates, kk), allow_masks=words)
            else:
                dev = torch.device(self._index.device)
                mat = torch.from_numpy(words.view(np.int32)).to(dev)
                index = torch.arange(len(pids), dtype=torch.int32, device=dev)
                ts, ti, tc = (np.asarray(t.cpu()) for t in self._index.search_pages(pids, kk, mat, index))
            t2 = time.perf_counter()
            out = [self._chunks(ts[i], ti[i], int(tc[i]), min_score) for i in range(len(pids))]
            t3 = time.perf_counter()
        self.last_query_timing = {"prepare_ms": (t1 - t0) * 1e3, "gpu_search_ms": (t2 - t1) * 1e3,
                                  "build_chunks_ms": (t3 - t2) * 1e3, "total_ms": (t3 - t0) * 1e3}
        if self._two_stage is not None:
            self.last_query_timing.update({k: float(v) for k, v in self._two_stage.last_timing_ms.items()})
        return out

    async def query_similar_with_feedback(self, query_embedding=None, k: int = 10,
                                          positive_chunks: Sequence[Tuple[str, int]] = (),
                                          negative_chunks: Sequence[Tuple[str, int]] = (),
                                          doc_ids: Optional[List[str]] = None, app_id: Optional[str] = None,
                                          min_score: Optional[float] = None) -> List[DocumentChunk]:
        """Relevance feedback (extension; the "recommend" call of vector databases): chunks like the query and the chunks
        marked good, unlike the chunks marked wrong.  Chunk ids follow ``get_chunks_by_id``'s rules (unknown or deleted
        chunks and chunks of another ``app_id`` are skipped, duplicates collapsed); a chunk in both lists is a ValueError.
        The query (if given) and each positive chunk weigh +1/n_pos, each negative chunk -1/n_neg, so a chunk's score is
        its mean similarity to the positives minus its mean similarity to the negatives, each on the page-to-page scale of
        query_similar_to_chunks (MaxSim per example row or query token: about 1 for an exact copy of unit-norm positives).
        ``doc_ids`` / ``app_id`` filter the results as in query_similar and the example chunks are never returned;
        ``min_score`` drops hits below it.  Every example shares one pass over the corpus (with a first stage, the
        positives' candidates); masks, GPU search and chunk construction are one critical section.  No query and no
        visible positive chunk: []."""
        q = None if query_embedding is None else as_query_matrix(query_embedding)
        pos_ids = list(dict.fromkeys((d, int(n)) for d, n in positive_chunks))
        neg_ids = list(dict.fromkeys((d, int(n)) for d, n in negative_chunks))
        both = set(pos_ids) & set(neg_ids)
        if both:
            raise ValueError(f"chunks named as both positive and negative examples: {sorted(both)}")
        if k <= 0 or (q is None and not pos_ids):
            return []
        return await asyncio.to_thread(self._feedback_locked, q, int(k), pos_ids, neg_ids, doc_ids, app_id, min_score)

    def _feedback_locked(self, q, k, pos_ids, neg_ids, doc_ids, app_id, min_score):
        import torch

        t0 = time.perf_counter()
        with self._lock:
            pos = [pid for pid, _ in self._visible_records(pos_ids, app_id)] if pos_ids else []
            neg = [pid for pid, _ in self._visible_records(neg_ids, app_id)] if neg_ids else []
            n_pos = len(pos) + (q is not None)
            if n_pos == 0:
                return []
            n = len(self.catalog)
            mask = self.catalog.allow_mask(doc_ids, app_id)
            mask = self.catalog.alive[:n].copy() if mask is None else mask
            mask[pos + neg] = False  # the examples themselves are never results
            if not mask.any():
                return []
            words = PageCatalog.mask_words(mask)[None]
            kk = min(_capped_k(k), n)
            queries = [] if q is None else [q]
            pages = pos + neg
            weights = [1.0 / n_pos] * n_pos + ([-1.0 / len(neg)] * len(neg) if neg else [])
            ex_req = [0] * len(weights)
            t1 = time.perf_counter()
            if self._two_stage is not None:  # the positives' first-stage candidates, under the same mask
                ts, ti, tc = self._two_stage.search_examples(queries, pages, ex_req, weights, 1, kk,
                                                             n_candidates=max(self._n_candidates, kk), allow_masks=words)
            else:
                dev = torch.device(self._index.device)
                q_dev = None if q is None else torch.from_numpy(np.ascontiguousarray(q, np.float32)).to(dev)
                mat = torch.from_numpy(words.view(np.int32)).to(dev)
                index = torch.zeros((1,), dtype=torch.int32, device=dev)
                ts, ti, tc = (np.asarray(t.cpu()) for t in self._index.search_examples(
                    q_dev, [int(q.shape[0])] if q is not None else [], pages, ex_req, weights, 1, kk, mat, index))
            t2 = time.perf_counter()
            out = self._chunks(ts[0], ti[0], int(tc[0]), min_score)
            t3 = time.perf_counter()
        self.last_query_timing = {"prepare_ms": (t1 - t0) * 1e3, "gpu_search_ms": (t2 - t1) * 1e3,
                                  "build_chunks_ms": (t3 - t2) * 1e3, "total_ms": (t3 - t0) * 1e3}
        if self._two_stage is not None:
            self.last_query_timing.update({k: float(v) for k, v in self._two_stage.last_timing_ms.items()})
        return out

    async def get_chunks_by_id(self, chunk_identifiers: List[Tuple[str, int]], app_id: Optional[str] = None,
                               skip_image_content: bool = False) -> List[DocumentChunk]:
        if not chunk_identifiers:
            return []
        return [_document_chunk(rec, 0.0) for _, rec in self._visible_records(chunk_identifiers, app_id)]

    def _visible_records(self, chunk_identifiers, app_id) -> List[Tuple[int, PageRecord]]:
        """(page id, record) of every live chunk named, in first-mention order, duplicates collapsed, skipping chunks stored
        under another app_id."""
        out = []
        for doc_id, chunk_num in dict.fromkeys((d, int(n)) for d, n in chunk_identifiers):
            pid = self.catalog.lookup(doc_id, chunk_num)
            if pid is None:
                continue
            rec = self.catalog.records[pid]
            if app_id is not None and rec.app_id is not None and rec.app_id != app_id:
                continue
            out.append((pid, rec))
        return out

    async def explain_chunks(self, query_embedding, chunk_identifiers: List[Tuple[str, int]], app_id: Optional[str] = None,
                             with_map: bool = False) -> List[Dict[str, Any]]:
        """Why chunks matched a query (extension): one record per visible chunk, under the rules of ``get_chunks_by_id``
        (unknown or deleted chunks and chunks of another ``app_id`` are skipped, duplicates collapsed), holding
        ``document_id``, ``chunk_number``, ``score`` (the sum of its token scores: the chunk's query_similar score),
        ``token_scores`` float32 [T], ``best_patch`` int32 [T] (per query token, the row of the chunk's embedding -- in the order
        the embedding model emitted it -- that answered it) and, with ``with_map``, ``sim_map`` float32 [T, n_rows].  Placing
        rows on the page image (patch grid, special tokens) is the embedding processor's business."""
        q = as_query_matrix(query_embedding)
        if not chunk_identifiers:
            return []
        return await asyncio.to_thread(self._explain_locked, q, list(chunk_identifiers), app_id, bool(with_map))

    def _explain_locked(self, q, chunk_identifiers, app_id, with_map):
        with self._lock:
            recs = self._visible_records(chunk_identifiers, app_id)
            if not recs:
                return []
            map_rows = max(rec.n_rows for _, rec in recs) if with_map else 0
            ts, br, sm = self._index.explain([q], [pid for pid, _ in recs], map_rows)
            ts, br = ts[0].cpu().numpy(), br[0].cpu().numpy()
            sm = sm[0].cpu().numpy() if sm is not None else None
        out = []
        for j, (_, rec) in enumerate(recs):
            r = {"document_id": rec.document_id, "chunk_number": rec.chunk_number, "score": float(ts[j].sum(dtype=np.float64)),
                 "token_scores": ts[j], "best_patch": br[j]}
            if with_map:
                r["sim_map"] = sm[j][:, :rec.n_rows]
            out.append(r)
        return out

    async def delete_chunks_by_document_id(self, document_id: str, app_id: Optional[str] = None) -> bool:
        try:  # off the event loop: the lock may be held by a GPU pass, and a compaction copies device memory
            await asyncio.to_thread(self._delete_locked, document_id)
            return True
        except Exception as e:  # noqa: BLE001  (reference returns False on error: multi_vector_store.py:949-951)
            logger.error("Error deleting chunks for document %s: %s", document_id, e)
            return False

    def _delete_locked(self, document_id: str) -> None:
        with self._lock:
            self.catalog.delete_document(document_id)
            if self._journal is not None:
                self._journal.log_delete(document_id)
            if self.catalog.dead_fraction > self.compact_dead_fraction:
                self._compact_locked()

    def _compact_locked(self):
        """Drop tombstoned pages: rebuild the device corpus from the surviving packed rows (device-to-device)."""
        keep, remap = self.catalog.compaction_plan()
        target = self._two_stage or self._index
        if hasattr(target, "compact"):
            target.compact(keep)
        self.catalog.apply_compaction(keep)
        if self._dup is not None:  # the pair table follows the pages: pairs with a dropped page go
            import torch

            d = self._dup
            m = torch.from_numpy(remap).to(d["a"].device)
            a, b = m[d["a"]], m[d["b"]]
            ok = (a >= 0) & (b >= 0)
            self._dup = {"a": a[ok].contiguous(), "b": b[ok].contiguous(), "sab": d["sab"][ok].contiguous(),
                         "sba": d["sba"][ok].contiguous(), "n_indexed": int((keep < d["n_indexed"]).sum())}

    # ------------------------------------------------------------------ persistence (SURVEY 8f-2)
    def save(self, directory: str) -> None:
        """Checkpoint: tombstoned pages are compacted away and the live corpus is written as ONE base segment of a journal
        directory (shardfile.StoreJournal); the legacy pair corpus.b2ms + catalog.jsonl is written too so that
        ``load`` of older callers keeps working."""
        import os

        from . import shardfile

        os.makedirs(directory, exist_ok=True)
        with self._lock:
            if self.catalog.dead_fraction > 0:
                self._compact_locked()
            shardfile.save_index(self._index, os.path.join(directory, "corpus.b2ms"))
            with open(os.path.join(directory, "catalog.jsonl"), "w") as f:
                for r in self.catalog.records:
                    f.write(json.dumps(dataclasses.asdict(r)) + "\n")
            if self._journal is not None and os.path.abspath(self._journal.dir) == os.path.abspath(directory):
                self._journal.reset()
                if len(self.catalog):
                    self._journal.log_add(self._index, 0, len(self.catalog), [dataclasses.asdict(r) for r in self.catalog.records],
                                          self._journal_rows(0, len(self.catalog)))

    @classmethod
    def load(cls, directory: str, device: int = 0, **kw) -> "B200MultiVectorStore":
        import os

        from . import shardfile

        index = shardfile.load_index(os.path.join(directory, "corpus.b2ms"), device=device, tier=kw.get("corpus_tier", "hbm"))
        store = cls(device=device, mode=index.dtype_name, auto_initialize=False, index=index, **kw)
        with open(os.path.join(directory, "catalog.jsonl")) as f:
            for line in f:
                store.catalog.add(PageRecord(**json.loads(line)))
        if len(store.catalog) != index.n_pages:
            raise ValueError("catalogue and shard file disagree on the page count")
        store.initialize()  # two-stage mode: rebuilds the FDE matrix from the packed rows; applies zero_pad_compat
        return store

    @classmethod
    def open(cls, directory: str, device: int = 0, mode: str = "bf16", **kw) -> "B200MultiVectorStore":
        """Durable store: replay ``directory``'s journal (segments appended by earlier store_embeddings calls, tombstones of
        earlier deletes -- fast_multivector_store.py:673-707 / multi_vector_store.py:929-933 persist the same two operations)
        and keep journaling.  Nothing is ever rewritten in place; ``save(directory)`` checkpoints."""
        from . import shardfile

        journal = shardfile.StoreJournal(directory)
        store = cls(device=device, mode=mode, **kw)
        ops = journal.read_ops()
        # size the block once, from the segment headers
        segs = [shardfile.read_header(journal.segment_files(op["seq"])[0])[0] for op in ops if op["op"] == "segment"]
        store._index.reserve_rows(sum(int(h["n_rows_padded"]) for h in segs))
        for op in ops:
            if op["op"] == "segment":
                seg, cat, fde = journal.segment_files(op["seq"])
                first = store._index.n_pages
                shardfile.load_index(seg, device=device, into=store._index)
                with open(cat) as f:
                    for line in f:
                        store.catalog.add(PageRecord(**json.loads(line)))
                if store._two_stage is not None:
                    store._two_stage.replay_segment(fde)
                if store._index.n_pages - first != int(op["pages"]) or len(store.catalog) != store._index.n_pages:
                    raise ValueError(f"{seg}: segment and journal disagree on the page count")
            elif op["op"] == "delete":
                store.catalog.delete_document(op["document_id"])
        if store._two_stage is not None:
            store._two_stage.replay_done()
        with store._lock:
            if store.catalog.dead_fraction > store.compact_dead_fraction:
                store._compact_locked()
        store._journal = journal
        return store
