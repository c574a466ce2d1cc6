"""Pairs of calls on one handle that the stream-order tests put in flight together (no GPU needed to import).

Every case names call A, left in flight on one stream, and call B, issued right after A returns: on a second stream, on
the handle's own stream (the *_host entry points, set_corpus*, fde_configure*), or -- for the controls -- on A's stream or
on a second handle.  tests/test_gpu_stream_order.py runs each case for each of its corpus kinds and requires both calls to
return, bit for bit, what they return when run alone; tests/test_stream_order_cpu.py requires every exported function of
include/b200ms.h that takes a stream or enqueues on the handle's stream to appear in some case.
"""
from __future__ import annotations

from dataclasses import dataclass
from typing import Tuple

# The calls a case can issue, and the exported functions each one runs, in order.
CALLS = {
    "search_device": ("b200ms_search_device",),
    "search_device_masked": ("b200ms_search_device_masked",),
    "search_host": ("b200ms_search_host",),
    "search_host_masked": ("b200ms_search_host_masked",),
    "rerank_device": ("b200ms_rerank_device",),
    "rerank_batch_device": ("b200ms_rerank_batch_device",),
    "explain_device": ("b200ms_explain_device",),
    "search_docs_device": ("b200ms_search_docs_device",),
    "rerank_docs_batch_device": ("b200ms_rerank_docs_batch_device",),
    # pack_queries -> score -> topk -> topk_docs over the caller's score matrix
    "score_topk": ("b200ms_pack_queries", "b200ms_score", "b200ms_topk", "b200ms_topk_docs"),
    "utilities": ("b200ms_sign_pack", "b200ms_hamming_batch", "b200ms_pack_pages", "b200ms_merge_topk",
                  "b200ms_bcast_device", "b200ms_allgather_topk"),
    # begin on A's stream; end (on A's stream) only after B has been issued
    "sharded_search": ("b200ms_sharded_search_begin", "b200ms_sharded_search_end"),
    # begin on the handle's stream; the blocking end only after B has been issued
    "sharded_search_host": ("b200ms_sharded_search_host_begin", "b200ms_sharded_search_host_end"),
    # query FDEs through the final projection (scratch fde_tmp), then the scan (scratch fde_q_bf16)
    "fde_encode_scan": ("b200ms_fde_encode", "b200ms_fde_scan"),
    # document FDEs of the attached corpus through the final projection, then finalize
    "fde_encode_corpus": ("b200ms_fde_encode_corpus", "b200ms_fde_finalize"),
    # another FDE configuration, then a query encoding under it
    "fde_configure": ("b200ms_fde_configure", "b200ms_fde_encode"),
    "fde_configure_ex": ("b200ms_fde_configure_ex", "b200ms_fde_encode"),
    # attach a different corpus to the same handle, then search it
    "set_corpus_search": ("b200ms_set_corpus", "b200ms_search_device"),
    "set_corpus_host_rerank": ("b200ms_set_corpus_host", "b200ms_rerank_batch_device"),
}

# Exports that take a stream but need more than one rank: nothing to put in flight on a one-GPU handle.
# tests/test_gpu_sharded_nccl.py runs them.
MULTI_RANK_ONLY = ("b200ms_send_device", "b200ms_recv_device")

# corpus kinds: (dtype of MaxSimIndex, option b1_tensor or None, tier)
KINDS = {
    "bf16": ("bf16", None, "hbm"),
    "int8": ("int8", None, "hbm"),
    "fp8": ("fp8", None, "hbm"),
    "b1_popc": ("binary", 0, "hbm"),
    "b1_wgmma": ("binary", 1, "hbm"),
    "bf16_host": ("bf16", None, "host"),
}


@dataclass(frozen=True)
class Case:
    name: str
    a: str
    b: str
    kinds: Tuple[str, ...]
    b_stream: str = "other"  # "other": a second stream; "same": A's stream (control)
    handles: int = 1         # 2: B runs on a second handle over the same rows, on its own stream (control)
    oracle: bool = False     # also check A's alone run against oracle.scoring


CASES = [
    Case("search_device-then-search_host", "search_device", "search_host",
         ("bf16", "int8", "fp8", "b1_popc", "b1_wgmma"), oracle=True),
    Case("search_device-then-masked", "search_device", "search_device_masked", ("bf16",)),
    Case("masked-then-search_host_masked", "search_device_masked", "search_host_masked", ("int8", "fp8")),
    Case("rerank_batch-then-rerank", "rerank_batch_device", "rerank_device", ("bf16", "int8")),
    Case("explain-then-rerank_batch", "explain_device", "rerank_batch_device", ("bf16", "fp8")),
    Case("search_docs-then-rerank_docs", "search_docs_device", "rerank_docs_batch_device", ("bf16", "b1_popc")),
    Case("score_topk-then-score_topk", "score_topk", "score_topk", ("fp8", "b1_popc", "b1_wgmma")),
    Case("search_device-then-utilities", "search_device", "utilities", ("bf16",)),
    Case("host_tier-rerank_batch-then-rerank", "rerank_batch_device", "rerank_device", ("bf16_host",)),
    Case("host_tier-rerank_batch-then-set_corpus_host", "rerank_batch_device", "set_corpus_host_rerank", ("bf16_host",)),
    Case("sharded-then-search_host", "sharded_search", "search_host", ("bf16",)),
    Case("sharded_host-then-search_device", "sharded_search_host", "search_device", ("int8",)),
    Case("fde_encode_corpus-then-fde_encode_scan", "fde_encode_corpus", "fde_encode_scan", ("bf16",)),
    Case("fde_encode_scan-then-fde_encode_scan", "fde_encode_scan", "fde_encode_scan", ("bf16",)),
    Case("fde_encode_scan-then-fde_configure", "fde_encode_scan", "fde_configure", ("bf16",)),
    Case("fde_encode_corpus-then-fde_configure_ex", "fde_encode_corpus", "fde_configure_ex", ("bf16",)),
    Case("search_device-then-set_corpus", "search_device", "set_corpus_search", ("bf16", "int8")),
    # controls: these never depended on the handle ordering its calls
    Case("control-same_stream", "search_device", "search_device_masked", ("bf16",), b_stream="same"),
    Case("control-two_handles", "search_device", "search_device", ("bf16",), handles=2),
]


def covered_exports():
    """Every exported function some case runs, as A or as B."""
    return {fn for c in CASES for call in (c.a, c.b) for fn in CALLS[call]}


def parametrize():
    """(case, kind) pairs and their test ids."""
    pairs = [(c, k) for c in CASES for k in c.kinds]
    return pairs, [f"{c.name}-{k}" for c, k in pairs]
