"""ShardedB200MultiVectorStore -- the BaseVectorStore plugin over all GPUs of one box (SURVEY 8e at the plugin level).

One process per GPU (torchrun).  Rank 0 is the process the Morphik API server talks to: it exposes the usual four async
methods (core/vector_store/base_vector_store.py:7-65).  Ranks > 0 call ``worker_loop()`` and execute the same command
stream.  Documents are assigned to ranks whole (least-loaded rank at first sight), so the ``doc_ids`` filter and
``delete_chunks_by_document_id`` stay rank-local and no page data ever moves between GPUs after ingest.

Command stream.  Every command is a FIXED 64-byte binary header (8 x int64: opcode, owner rank, item count, row count,
payload bytes, k, n_q, reserved) broadcast from rank 0, followed -- only when the header says so -- by one JSON payload
broadcast (document / app ids, page lengths, per-query filters).  Ingest rows go to the OWNING rank only (point-to-point
send/recv; rank 0 keeps them when it is the owner), query rows are broadcast.  After executing a command every rank
contributes a status word to one small all-reduce, so a failure on any rank (allocation, validation) becomes an exception
on rank 0 instead of a hang, and the worker loops stay alive.

Concurrent query_similar coroutines are coalesced on rank 0 (store.QueryCoalescer) into one command per GPU pass.
A query command: every rank builds its own page masks (one row per distinct (doc_ids, app_id) filter), scans its shard and
selects its top-k with GLOBAL ids ``(rank << 40) | local_page`` straight into the exchange layout -> ONE NCCL all-gather of
n_q*k*12 bytes per rank inside libb200ms -> merge on every rank (``ShardedMaxSim``) -> rank 0 turns ids into DocumentChunks.
With ``fde_candidates=N`` every rank runs the two-stage search of the "morphik" provider on its shard (FDE scan -> top-N
-> batched MaxSim rerank, fast_multivector_store.py:521-557) before the same single exchange.
Rank 0 mirrors every rank's catalogue (payloads and metadata live only there); mirror and index change together, inside
the command execution and under one lock, so their orders can never diverge.

The index factory and the collective helpers are injectable so the host logic runs under ``gloo`` on CPU with
oracle-backed stand-ins (tests/test_sharded_store_gloo.py); the product wiring is MaxSimIndex + NCCL.
"""
from __future__ import annotations

import asyncio
import json
import logging
import threading
from typing import Any, Callable, Dict, List, Optional, Sequence, Tuple

import numpy as np
import torch
import torch.distributed as dist

from .catalog import PageCatalog, PageRecord
from .models import DocumentChunk
from .sharded import ShardedMaxSim, exchange_bytes, exchange_views, gathered_candidates
from .store import BaseVectorStore, QueryCoalescer, _document_chunk, _QueryRequest, as_query_matrix, build_store_metrics

logger = logging.getLogger(__name__)
RANK_SHIFT = 40
OP_ADD, OP_QUERY, OP_DELETE, OP_STOP = 1, 2, 3, 4
HEADER_WORDS = 8
MAX_K = 4096
MERGE_CAPACITY = 8192  # candidates b200ms_merge_topk can sort per query: world * k must fit


def split_global_id(gid: int) -> Tuple[int, int]:
    return int(gid) >> RANK_SHIFT, int(gid) & ((1 << RANK_SHIFT) - 1)


class ShardedStoreError(RuntimeError):
    """A command failed on at least one rank (the message names the ranks); the store stays usable."""


class ShardedB200MultiVectorStore(QueryCoalescer, BaseVectorStore):
    def __init__(self, mode: str = "bf16", device: Optional[int] = None, group: Optional[dist.ProcessGroup] = None,
                 index_factory: Optional[Callable[[], Any]] = None, compact_dead_fraction: float = 0.3,
                 coalesce_queries: bool = True, max_coalesced_tokens: int = 1024, max_coalesced_queries: int = 64,
                 fde_candidates: Optional[int] = None):
        if not dist.is_initialized():
            raise RuntimeError("ShardedB200MultiVectorStore needs an initialised torch.distributed process group (torchrun)")
        self.group = group
        self.rank = dist.get_rank(group)
        self.world = dist.get_world_size(group)
        self.mode = mode
        self.uri = f"b200-sharded://{self.world}"
        self.storage = None
        self.compact_dead_fraction = float(compact_dead_fraction)
        self.fde_candidates = fde_candidates
        self._two_stage = None
        if index_factory is None:
            from .index import MaxSimIndex  # CUDA product path; raises without a GPU

            dev = self.rank if device is None else int(device)
            if fde_candidates:
                from .fde import TwoStageIndex

                self._two_stage = TwoStageIndex(device=dev, dtype=mode)
                index_factory = lambda: self._two_stage.index  # noqa: E731
            else:
                index_factory = lambda: MaxSimIndex(device=dev, dtype=mode)  # noqa: E731
        self.index = index_factory()
        self.data_device = getattr(self.index, "device", torch.device("cpu"))
        # catalogue of THIS rank's pages (rank 0 additionally mirrors everybody's, with payloads)
        self.catalogs: Dict[int, PageCatalog] = {r: PageCatalog() for r in (range(self.world) if self.rank == 0 else [self.rank])}
        self.doc_rank: Dict[str, int] = {}
        self.rank_rows = [0] * self.world
        self._lock = threading.RLock()  # re-entrant: a query holds it across the command AND the catalogue look-ups
        if hasattr(self.index, "sharded_search_begin"):  # CUDA index: the collective lives inside libb200ms
            self._sharded = ShardedMaxSim.from_index(self.index, id_base=self.rank << RANK_SHIFT, group=group)
        else:  # injected stand-in (CPU tests): same exchange layout over torch.distributed
            self._sharded = ShardedMaxSim(self._local_search_into, self._merge_gathered, group)
        self._init_coalescer(coalesce_queries, max_coalesced_tokens, max_coalesced_queries)
        self._mask_matrix: Optional[torch.Tensor] = None  # [n_distinct_filters, words] int32, this rank's pages
        self._mask_index: Optional[torch.Tensor] = None   # int32 [n_q]: row of _mask_matrix per query, -1 = unfiltered
        self.last_query_timing: Dict[str, float] = {}
        self._pending_payloads = None
        self._stage_events = None

    # ------------------------------------------------------------------ collective plumbing
    def _src(self) -> int:
        return dist.get_global_rank(self.group, 0) if self.group is not None else 0

    def _peer(self, r: int) -> int:
        return dist.get_global_rank(self.group, r) if self.group is not None else r

    def _bcast_header(self, words: Optional[Sequence[int]]) -> List[int]:
        t = torch.zeros(HEADER_WORDS, dtype=torch.int64, device=self.data_device)
        if self.rank == 0:
            t.copy_(torch.tensor(list(words) + [0] * (HEADER_WORDS - len(words)), dtype=torch.int64))
        dist.broadcast(t, src=self._src(), group=self.group)
        return [int(x) for x in t.cpu().tolist()]

    def _bcast_payload(self, obj: Any, n_bytes: int) -> Any:
        t = torch.empty(n_bytes, dtype=torch.uint8, device=self.data_device)
        if self.rank == 0 and n_bytes:
            t.copy_(torch.frombuffer(bytearray(obj), dtype=torch.uint8))
        if n_bytes:
            dist.broadcast(t, src=self._src(), group=self.group)
        return json.loads(bytes(t.cpu().numpy().tobytes()).decode()) if n_bytes else None

    def _bcast_rows(self, rows: Optional[np.ndarray], n_rows: int) -> torch.Tensor:
        t = torch.empty((n_rows, 128), dtype=torch.float32, device=self.data_device)
        if self.rank == 0:
            t.copy_(torch.from_numpy(np.ascontiguousarray(rows, dtype=np.float32)))
        if n_rows:
            if hasattr(self.index, "bcast") and self.world > 1:
                self.index.bcast(t, root=0)  # ncclBroadcast on the handle's communicator
            else:
                dist.broadcast(t, src=self._src(), group=self.group)
        return t

    def _rows_to_owner(self, rows: Optional[np.ndarray], n_rows: int, owner: int) -> Optional[torch.Tensor]:
        """Ingest rows travel to the owner only (the other ranks never see them): ncclSend / ncclRecv on the handle's own
        communicator with the CUDA index, torch.distributed send / recv with an injected stand-in (CPU tests)."""
        native = hasattr(self.index, "send")
        if self.rank == 0:
            t = torch.from_numpy(np.ascontiguousarray(rows, dtype=np.float32)).to(self.data_device)
            if owner != 0 and n_rows:
                if native:
                    self.index.send(t, owner)
                    torch.cuda.current_stream(self.data_device).synchronize()  # t dies with this frame
                else:
                    dist.send(t, dst=self._peer(owner), group=self.group)
            return t if owner == 0 else None
        if owner != self.rank:
            return None
        t = torch.empty((n_rows, 128), dtype=torch.float32, device=self.data_device)
        if n_rows:
            if native:
                self.index.recv(t, 0)
            else:
                dist.recv(t, src=self._src(), group=self.group)
        return t

    def _agree(self, err: Optional[BaseException]) -> None:
        """One all-reduce of a status bitmask after every command: rank r sets bit r when its part failed."""
        flag = torch.tensor([0 if err is None else (1 << self.rank)], dtype=torch.int64, device=self.data_device)
        dist.all_reduce(flag, op=dist.ReduceOp.SUM, group=self.group)  # distinct bits per rank: the sum is the OR
        bad = int(flag.item())
        if bad:
            ranks = [r for r in range(self.world) if bad >> r & 1]
            raise ShardedStoreError(f"command failed on rank(s) {ranks}" + (f": {err!r}" if err is not None else ""))

    # injected (stand-in) path: index.search_device / index.merge_topk behind the exchange layout
    def _local_search_into(self, q, q_lens, k, ids_view, scores_view):
        cat = self.catalogs[self.rank]
        if len(cat) == 0:
            ids_view.fill_(-1)
            scores_view.fill_(float("-inf"))
            return
        if self._mask_matrix is None:
            ts, ti, _ = self.index.search_device(q, list(q_lens), k, id_base=self.rank << RANK_SHIFT)
        else:
            ts, ti, _ = self.index.search_device(q, list(q_lens), k, allow_mask_dev=self._mask_matrix,
                                                 id_base=self.rank << RANK_SHIFT, mask_index_dev=self._mask_index)
        ids_view.copy_(ti)
        scores_view.copy_(ts)

    def _merge_gathered(self, gathered, world, n_q, k):
        ci, cs = gathered_candidates(gathered, world, n_q, k)
        return self.index.merge_topk(cs, ci, k)

    # ------------------------------------------------------------------ command execution (identical on every rank)
    def _build_masks(self, filters) -> None:
        cat = self.catalogs[self.rank]
        n = len(cat)
        masks = []
        for doc_ids, app_id in filters:
            visible, words = cat.allow_words(doc_ids, app_id) if n else (False, None)
            if not visible:  # nothing authorised on this rank: an all-zero mask keeps the query out of the local top-k
                words = np.zeros((n + 31) // 32, dtype=np.uint32)
            masks.append(words)
        mat, index = PageCatalog.stack_masks(masks)
        if mat is not None and n:
            self._mask_matrix = torch.from_numpy(mat.view(np.int32)).to(self.data_device)
            self._mask_index = torch.tensor(index, dtype=torch.int32, device=self.data_device)
        else:
            self._mask_matrix = self._mask_index = None

    def _two_stage_search(self, q: torch.Tensor, q_lens, k: int):
        """Per-rank two-stage search written into the exchange layout, then the one all-gather + merge (b200ms_allgather_topk)."""
        n_q = len(q_lens)
        xchg = torch.empty(exchange_bytes(n_q, k), dtype=torch.uint8, device=self.data_device)
        ids_v, sc_v = exchange_views(xchg, n_q, k)
        off = np.concatenate([[0], np.cumsum(q_lens)])
        queries = [q[int(off[i]):int(off[i + 1])] for i in range(n_q)]
        mask = None
        if self._mask_matrix is not None:
            if self._mask_matrix.shape[0] != 1 or bool((self._mask_index != 0).any()):
                raise ValueError("two-stage mode takes one filter per pass (coalescing is off in this mode)")
            mask = self._mask_matrix[0].contiguous()
        if self._two_stage.n_pages == 0:
            ids_v.fill_(-1)
            sc_v.fill_(float("-inf"))
        else:
            kk = min(k, self._two_stage.n_pages)
            ts, ti, _, ev = self._two_stage.search_device(queries, kk, max(int(self.fde_candidates), kk), mask,
                                                          id_base=self.rank << RANK_SHIFT)
            ids_v.fill_(-1)
            sc_v.fill_(float("-inf"))
            ids_v[:, : ti.shape[1]].copy_(ti)
            sc_v[:, : ts.shape[1]].copy_(ts)
            self._stage_events = ev
        return self.index.allgather_topk(xchg, n_q, k)

    def _execute(self, hdr: List[int], payload: Any, rows: Optional[np.ndarray]) -> Any:
        op = hdr[0]
        if op == OP_ADD:
            owner, n_items, n_rows = hdr[1], hdr[2], hdr[3]
            recs, lens = payload["recs"], payload["lens"]
            mine = self._rows_to_owner(rows, n_rows, owner)
            err = None
            try:  # phase 1: the only step that can fail -- the owner packs the pages into its shard
                if owner == self.rank:
                    off = np.concatenate([[0], np.cumsum(lens)]).astype(np.int64)
                    (self._two_stage or self.index).add_pages([mine[off[i]:off[i + 1]] for i in range(n_items)])
            except Exception as e:  # noqa: BLE001  (reported through _agree; the collective stream stays in step)
                err = e
            self._agree(err)  # raises on every rank if the owner failed: nobody has touched its bookkeeping yet
            # phase 2: bookkeeping, identical on every rank and in command-stream order (rank 0's mirror included)
            for (doc, _num, _app) in recs:
                self.doc_rank[doc] = owner
            self.rank_rows[owner] += int(sum(lens))
            if owner in self.catalogs:
                extra = self._pending_payloads if self.rank == 0 else None
                for i, ((doc, num, app), n) in enumerate(zip(recs, lens)):
                    content, meta = extra[i] if extra is not None else ("", {})
                    self.catalogs[owner].add(PageRecord(doc, int(num), content, meta, app, int(n)))
            return None
        if op == OP_QUERY:
            k, n_q, n_rows = hdr[5], hdr[6], hdr[3]
            q_lens, filters = payload["q_lens"], [(f[0], f[1]) for f in payload["filters"]]
            q = self._bcast_rows(rows, n_rows)
            err, out = None, None
            try:
                self._build_masks(filters)
            except Exception as e:  # noqa: BLE001
                err = e
            self._agree(err)  # nobody enters the collective search unless every rank could build its masks
            if self._two_stage is not None:
                return self._two_stage_search(q, q_lens, k)
            return self._sharded.search(q, q_lens, k, self._mask_matrix, self._mask_index)
        if op == OP_DELETE:
            document_id = payload["document_id"]
            err, found = None, False
            try:
                owner = self.doc_rank.pop(document_id, None)
                found = owner is not None
                cat = self.catalogs.get(owner) if found else None  # rank 0 mirrors every rank; rank r only knows its own shard
                if cat is not None:
                    freed = sum(cat.records[p].n_rows for p in cat.pages_of(document_id))
                    cat.delete_document(document_id)
                    self.rank_rows[owner] -= freed
                    if cat.dead_fraction > self.compact_dead_fraction:  # same decision on the owner and on rank 0's mirror
                        keep, _ = cat.compaction_plan()
                        if owner == self.rank:
                            (self._two_stage or self.index).compact(keep)
                        cat.apply_compaction(keep)
            except Exception as e:  # noqa: BLE001
                err = e
            self._agree(err)
            return found
        if op == OP_STOP:
            return "stop"
        raise ValueError(f"unknown opcode {op}")

    def worker_loop(self) -> None:
        """Ranks > 0: execute rank 0's command stream until close().  A failing command is reported to rank 0 through the
        status all-reduce and the loop keeps serving."""
        assert self.rank != 0, "rank 0 drives the store through the BaseVectorStore methods"
        while True:
            hdr = self._bcast_header(None)
            payload = self._bcast_payload(None, hdr[4])
            try:
                if self._execute(hdr, payload, None) == "stop":
                    if hasattr(self.index, "close"):
                        self.index.close()  # releases this rank's communicator alongside rank 0's close()
                    return
            except ShardedStoreError as e:
                logger.error("sharded store command failed: %s", e)

    def _drive(self, hdr: List[int], payload_obj: Any = None, rows: Optional[np.ndarray] = None, payloads=None) -> Any:
        """Rank 0: publish a command (header, JSON payload) and execute it locally -- one critical section, so the command
        stream, the index and every catalogue (mirrors included) advance together."""
        with self._lock:
            blob = json.dumps(payload_obj).encode() if payload_obj is not None else b""
            hdr = list(hdr) + [0] * (HEADER_WORDS - len(hdr))
            hdr[4] = len(blob)
            self._pending_payloads = payloads
            self._bcast_header(hdr)
            payload = self._bcast_payload(blob, len(blob))
            try:
                return self._execute(hdr, payload, rows)
            finally:
                self._pending_payloads = None

    # ------------------------------------------------------------------ BaseVectorStore surface (rank 0)
    def initialize(self) -> bool:
        return True

    def close(self) -> None:
        if self.rank == 0 and dist.is_initialized():
            self._drive([OP_STOP])
        if hasattr(self.index, "close"):
            self.index.close()

    def _add_document_locked(self, doc: str, items, app_id) -> None:
        """Owner choice, mirror update and index update in ONE critical section (command-stream order)."""
        with self._lock:
            owner = self.doc_rank.get(doc)
            if owner is None:
                owner = int(np.argmin(self.rank_rows))  # whole documents go to the least-loaded rank
            lens = [int(e.shape[0]) for _, e in items]
            recs = [(c.document_id, int(c.chunk_number), app_id) for c, _ in items]
            rows = np.concatenate([e for _, e in items]) if sum(lens) else np.zeros((0, 128), np.float32)
            payloads = [(c.content, dict(c.metadata or {})) for c, _ in items]
            self._drive([OP_ADD, owner, len(items), int(sum(lens))], {"recs": recs, "lens": lens}, rows, payloads)

    async def store_embeddings(self, chunks: List[DocumentChunk], app_id: Optional[str] = None
                               ) -> Tuple[bool, List[str], Dict[str, Any]]:
        assert self.rank == 0
        by_doc: Dict[str, List[Tuple[DocumentChunk, np.ndarray]]] = {}
        for c in chunks:
            if getattr(c, "embedding", None) is None:
                logger.error("Missing embeddings for chunk %s-%s", c.document_id, c.chunk_number)
                continue
            emb = np.asarray(c.embedding.detach().float().cpu().numpy() if hasattr(c.embedding, "detach") else c.embedding,
                             dtype=np.float32)
            if emb.ndim == 1:
                emb = emb[None, :]
            if emb.ndim != 2 or emb.shape[1] != 128:
                raise ValueError(f"chunk {c.document_id}-{c.chunk_number}: embedding must be [P,128], got {tuple(emb.shape)}")
            by_doc.setdefault(c.document_id, []).append((c, emb))
        ids: List[str] = []
        for doc, items in by_doc.items():
            await asyncio.to_thread(self._add_document_locked, doc, items, app_id)
            ids.extend(f"{c.document_id}-{c.chunk_number}" for c, _ in items)
        return True, ids, build_store_metrics(vector_store_rows=len(ids), vector_store_backend=f"b200-hbm x{self.world}")

    async def query_similar(self, query_embedding, k: int, doc_ids: Optional[List[str]] = None,
                            app_id: Optional[str] = None, skip_image_content: bool = False) -> List[DocumentChunk]:
        assert self.rank == 0
        q = as_query_matrix(query_embedding)
        if k <= 0 or all(len(c) == 0 for c in self.catalogs.values()):
            return []
        if self.coalesce_queries and self._two_stage is None:
            return await self._enqueue_query(q, k, doc_ids, app_id)
        return (await asyncio.to_thread(self._search_coalesced_locked, [_QueryRequest(q, int(k), doc_ids, app_id, None)]))[0]

    def _search_coalesced_locked(self, batch) -> List[List[DocumentChunk]]:
        """One command (= one pass on every GPU) for a batch of independent requests."""
        import time

        t0 = time.perf_counter()
        q_lens = [int(r.q.shape[0]) for r in batch]
        cap = max(1, min(MAX_K, MERGE_CAPACITY // self.world))  # world * k candidates must fit the merge
        kmax = max(r.k for r in batch)
        if kmax > cap:
            logger.warning("k=%d exceeds the sharded store's limit of %d per query (world=%d); truncated", kmax, cap, self.world)
        kk = max(1, min(int(kmax), cap))
        rows = np.concatenate([r.q for r in batch]) if len(batch) > 1 else batch[0].q
        out = []
        with self._lock:
            filters = [[None if r.doc_ids is None else list(r.doc_ids), r.app_id] for r in batch]
            ts, ti, tc = self._drive([OP_QUERY, 0, 0, int(sum(q_lens)), 0, kk, len(batch)], {"q_lens": q_lens, "filters": filters}, rows)
            ts, ti, tc = ts.cpu().numpy(), ti.cpu().numpy(), tc.cpu().numpy()
            t1 = time.perf_counter()
            for i, r in enumerate(batch):
                hits = []
                for j in range(min(int(tc[i]), r.k)):
                    rk, local = split_global_id(ti[i, j])
                    hits.append(_document_chunk(self.catalogs[rk].records[local], ts[i, j]))
                out.append(hits)
        t2 = time.perf_counter()
        self.last_query_timing = {"coalesced_queries": float(len(batch)), "gpu_search_ms": (t1 - t0) * 1e3,
                                  "build_chunks_ms": (t2 - t1) * 1e3, "total_ms": (t2 - t0) * 1e3}
        ev = self._stage_events
        if self._two_stage is not None and ev is not None:  # the reference's stage names (fast_multivector_store.py:523-605)
            self.last_query_timing.update(self._two_stage.stage_timing_ms(ev), load_contents_ms=0.0)
        return out

    async def get_chunks_by_id(self, chunk_identifiers: List[Tuple[str, int]], app_id: Optional[str] = None,
                               skip_image_content: bool = False) -> List[DocumentChunk]:
        assert self.rank == 0
        out = []
        with self._lock:
            for doc_id, num in dict.fromkeys((d, int(n)) for d, n in chunk_identifiers):
                r = self.doc_rank.get(doc_id)
                pid = None if r is None else self.catalogs[r].lookup(doc_id, num)
                if pid is None:
                    continue
                rec = self.catalogs[r].records[pid]
                if app_id is not None and rec.app_id is not None and rec.app_id != app_id:
                    continue
                out.append(_document_chunk(rec, 0.0))
        return out

    async def index_duplicates(self, *args, **kw):
        """Not supported: duplicate detection runs on one HBM-tier store (B200MultiVectorStore.index_duplicates)."""
        raise NotImplementedError("the sharded store has no duplicate detection; use B200MultiVectorStore")

    async def find_duplicate_chunks(self, *args, **kw):
        """Not supported (see index_duplicates)."""
        raise NotImplementedError("the sharded store has no duplicate detection; use B200MultiVectorStore")

    async def query_similar_distinct(self, *args, **kw):
        """Not supported (see index_duplicates)."""
        raise NotImplementedError("the sharded store has no duplicate detection; use B200MultiVectorStore")

    async def delete_chunks_by_document_id(self, document_id: str, app_id: Optional[str] = None) -> bool:
        assert self.rank == 0
        try:
            await asyncio.to_thread(self._drive, [OP_DELETE], {"document_id": document_id})
            return True
        except Exception as e:  # noqa: BLE001
            logger.error("Error deleting chunks for document %s: %s", document_id, e)
            return False
