"""Document-sharded MaxSim search over the GPUs of one box (SURVEY 8e).

Every page's score is independent of every other page, so the corpus partitions by document: rank r owns a contiguous
range of whole documents (balanced by patch rows, optionally weighted by each GPU's measured scan rate), scans only its
shard, and the ranks exchange nothing but their per-query top-k lists: ONE NCCL all-gather of ``n_q * k * 12`` bytes per
rank (int64 global page id + float32 score), followed by a merge on every rank.  No page data ever crosses NVLink.  The
reference has nothing comparable (it is a single-process asyncio server); this is the multi-GPU extension the north star
asks for.

Product wiring (``ShardedMaxSim.from_index``): the collective lives INSIDE libb200ms (``b200ms_comm_init`` +
``b200ms_sharded_search_begin/_end``, csrc/comm.cu) -- the local top-k is written straight into the exchange layout, NCCL
gathers it on the handle's communication stream and ``merge_topk_kernel`` reads the gathered layout in place, so a query
step issues no torch op at all.  ``begin`` / ``end`` expose the two-slot pipeline: the scan of step i+1 starts without
waiting for the slowest rank's step i.

Test wiring: the local search and the merge are injectable and the exchange then runs over ``torch.distributed`` (any
backend), so the host logic -- shard plan, exchange layout, gather, merge order -- is testable on CPU with ``gloo``
(tests/test_sharded_gloo.py).
"""
from __future__ import annotations

from typing import Callable, List, Optional, Sequence, Tuple

import torch
import torch.distributed as dist


def plan_document_shards(doc_rows: Sequence[int], world: int, weights: Optional[Sequence[float]] = None
                         ) -> List[Tuple[int, int]]:
    """Split documents 0..D-1 (doc_rows[d] = patch rows of document d) into `world` contiguous ranges whose row totals
    are proportional to ``weights`` (default: equal -- pass each rank's measured scan rate to give a GPU that runs slower
    under its power cap a smaller shard).  Returns [(doc_begin, doc_end)] per rank; ranges may be empty when D < world."""
    total = int(sum(int(x) for x in doc_rows))
    w = [1.0] * world if weights is None else [float(x) for x in weights]
    if len(w) != world or any(x <= 0 for x in w):
        raise ValueError("weights: one positive number per rank")
    wsum = sum(w)
    bounds = [0]
    acc = 0
    d = 0
    n = len(doc_rows)
    cum = 0.0
    for r in range(1, world):
        cum += w[r - 1]
        target = total * cum / wsum
        while d < n and acc + int(doc_rows[d]) / 2.0 <= target:
            acc += int(doc_rows[d])
            d += 1
        bounds.append(d)
    bounds.append(n)
    return [(bounds[r], bounds[r + 1]) for r in range(world)]


# ---- the exchange layout (same bytes as include/b200ms.h "xchg"): [n_q*k int64 ids][n_q*k float32 scores]
def exchange_bytes(n_q: int, k: int) -> int:
    """= b200ms_xchg_bytes: 12 bytes per entry, padded to 16 so that every rank's block of the gathered buffer is aligned."""
    return (int(n_q) * int(k) * 12 + 15) // 16 * 16


def exchange_views(buf: torch.Tensor, n_q: int, k: int) -> Tuple[torch.Tensor, torch.Tensor]:
    """uint8 [n_q*k*12] -> (ids int64 [n_q,k], scores float32 [n_q,k]) views of the same memory: the local top-k is written
    in place, nothing is packed or copied before the collective."""
    n = n_q * k
    return buf[: n * 8].view(torch.int64).view(n_q, k), buf[n * 8: n * 12].view(torch.float32).view(n_q, k)


def gathered_candidates(gathered: torch.Tensor, world: int, n_q: int, k: int) -> Tuple[torch.Tensor, torch.Tensor]:
    """[world * n_q*k*12] uint8 -> candidate ids [n_q, world*k] and scores [n_q, world*k] (rank-major), for host-side merges
    (the CUDA merge reads the gathered buffer directly)."""
    g = gathered.view(world, exchange_bytes(n_q, k))
    n = n_q * k
    ids = g[:, : n * 8].contiguous().view(torch.int64).view(world, n_q, k)
    sc = g[:, n * 8: n * 12].contiguous().view(torch.float32).view(world, n_q, k)
    return (ids.permute(1, 0, 2).reshape(n_q, world * k).contiguous(), sc.permute(1, 0, 2).reshape(n_q, world * k).contiguous())


LocalSearchInto = Callable[[torch.Tensor, Sequence[int], int, torch.Tensor, torch.Tensor], None]
MergeGathered = Callable[[torch.Tensor, int, int, int], Tuple[torch.Tensor, torch.Tensor, torch.Tensor]]


class ShardedMaxSim:
    """Per-rank object: local shard search + all-gather + merge.  ``search`` returns the same result on every rank."""

    def __init__(self, local_search_into: Optional[LocalSearchInto] = None, merge_gathered: Optional[MergeGathered] = None,
                 group: Optional[dist.ProcessGroup] = None, index=None, id_base: int = 0):
        self.local_search_into = local_search_into
        self.merge_gathered = merge_gathered
        self.group = group
        self.index = index  # product path: a MaxSimIndex whose handle owns the NCCL communicator
        self.id_base = int(id_base)
        self.world = dist.get_world_size(group) if dist.is_initialized() else 1
        self.rank = dist.get_rank(group) if dist.is_initialized() else 0
        self._out = {}

    @classmethod
    def from_index(cls, index, id_base: int, group: Optional[dist.ProcessGroup] = None) -> "ShardedMaxSim":
        """Product wiring: `index` is this rank's MaxSimIndex over its shard; id_base = global id of its first page.
        Creates the handle's own NCCL communicator (torch.distributed only ships the 128-byte unique id, once)."""
        self = cls(group=group, index=index, id_base=id_base)
        if self.world > 1:
            dev = index.device
            uid = torch.zeros(128, dtype=torch.uint8, device=dev)
            if self.rank == 0:
                uid.copy_(torch.frombuffer(bytearray(index.comm_unique_id()), dtype=torch.uint8))
            dist.broadcast(uid, src=dist.get_global_rank(group, 0) if group is not None else 0, group=group)
            index.comm_init(bytes(uid.cpu().numpy().tobytes()), self.rank, self.world)
        else:
            index.comm_init(b"\0" * 128, 0, 1)
        return self

    def broadcast_queries(self, q: torch.Tensor, src: int = 0) -> torch.Tensor:
        if self.world > 1:
            if self.index is not None:
                self.index.bcast(q, root=src)  # ncclBroadcast on the handle's communicator
            else:
                dist.broadcast(q, src=src, group=self.group)
        return q

    # ------------------------------------------------------------------ pipelined form (product path only)
    def begin(self, q: torch.Tensor, q_lens: Sequence[int], k: int, out=None, allow_masks_dev=None, mask_index_dev=None):
        """Enqueue this rank's scan + top-k and, behind it on the communication stream, the all-gather + merge.  Returns
        (ticket, (scores, ids, counts)); the tensors are valid after ``end(ticket)``.  At most two tickets in flight."""
        if self.index is None:
            raise RuntimeError("begin/end need the CUDA index (ShardedMaxSim.from_index)")
        from .index import _topk_outputs

        out = _topk_outputs(len(q_lens), k, self.index.device, out)
        t = self.index.sharded_search_begin(q, q_lens, k, self.id_base, out, allow_masks_dev, mask_index_dev)
        return t, out

    def end(self, ticket: int) -> None:
        self.index.sharded_search_end(ticket)

    # ------------------------------------------------------------------ synchronous form
    def search(self, q: torch.Tensor, q_lens: Sequence[int], k: int, allow_masks_dev=None, mask_index_dev=None):
        """q: [sum T,128] on this rank's device (identical on all ranks -- see broadcast_queries).
        Returns (scores [n_q,k], global page ids [n_q,k], counts [n_q])."""
        n_q = len(q_lens)
        if self.index is not None:
            t, out = self.begin(q, q_lens, k, None, allow_masks_dev, mask_index_dev)
            self.end(t)
            return out
        # injected path (CPU tests): same exchange layout, torch.distributed as the transport
        mine = torch.empty(exchange_bytes(n_q, k), dtype=torch.uint8, device=q.device)
        ids_v, sc_v = exchange_views(mine, n_q, k)
        self.local_search_into(q, q_lens, k, ids_v, sc_v)
        if self.world == 1:
            return self.merge_gathered(mine, 1, n_q, k)
        gathered = torch.empty(self.world * mine.numel(), dtype=torch.uint8, device=mine.device)
        dist.all_gather_into_tensor(gathered, mine, group=self.group)  # the one collective of the path
        return self.merge_gathered(gathered, self.world, n_q, k)
