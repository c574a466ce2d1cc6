"""Every Python entry point that hands device tensors to libb200ms refuses a tensor the library would misread -- an allow
mask shorter than the corpus, float16 queries, fewer query rows than sum(q_lens), result buffers of the wrong shape --
with ValueError, before any kernel is launched."""
import numpy as np
import pytest

pytestmark = pytest.mark.gpu

torch = pytest.importorskip("torch")
if not torch.cuda.is_available():  # pragma: no cover
    pytest.skip("CUDA device required", allow_module_level=True)

from morphik_core_b200.fde import TwoStageIndex  # noqa: E402
from morphik_core_b200.index import MaxSimIndex  # noqa: E402

N_PAGES, K = 70, 5  # 70 pages: 3 mask words
LENS = [20, 12]


def _pages(rng):
    return [rng.standard_normal((int(n), 128)).astype(np.float32) for n in rng.integers(1, 60, size=N_PAGES)]


def _refused(index, calls):
    before = index.launch_count()
    for what, call in calls:
        with pytest.raises(ValueError):
            call()
        assert index.launch_count() == before, what


def test_index_entry_points_refuse_bad_tensors():
    rng = np.random.default_rng(3)
    idx = MaxSimIndex(dtype="bf16")
    idx.add_pages(_pages(rng))
    dev = idx.device
    n_q = len(LENS)
    q = torch.from_numpy(rng.standard_normal((sum(LENS), 128)).astype(np.float32)).to(dev)
    q16, q_short = q.half(), q[:-1]
    mask, short_mask = torch.full((3,), -1, dtype=torch.int32, device=dev), torch.full((2,), -1, dtype=torch.int32, device=dev)
    mat, short_mat = mask.view(1, 3), short_mask.view(1, 2)
    mi = torch.zeros(n_q, dtype=torch.int32, device=dev)
    out = tuple(torch.empty(s, dtype=d, device=dev) for s, d in (((n_q, K), torch.float32), ((n_q, K), torch.int64),
                                                                  ((n_q,), torch.int32)))
    wide = tuple(torch.empty(s, dtype=d, device=dev) for s, d in (((n_q, K + 1), torch.float32), ((n_q, K + 1), torch.int64),
                                                                   ((n_q,), torch.int32)))
    cand = torch.arange(8, dtype=torch.int64, device=dev)
    cand2 = cand.repeat(n_q, 1)
    page_doc = torch.arange(N_PAGES, dtype=torch.int32, device=dev)
    idx.comm_init(b"\0" * 128, 0, 1)

    # the valid calls work (and attach the corpus, so that the refused ones below have nothing left to prepare)
    idx.search_device(q, LENS, K, mask, out=out)
    idx.search_device(q, LENS, K, mat, mask_index_dev=mi)
    idx.rerank(q, LENS, cand, K)
    idx.rerank_batch(q, LENS, cand2, K)
    idx.search_docs_device(q, LENS, K, 2, page_doc, N_PAGES, mask)
    idx.rerank_docs_batch(q, LENS, cand2, K, 2, page_doc, N_PAGES)
    idx.sharded_search_end(idx.sharded_search_begin(q, LENS, K, 0, out, mat, mi))
    torch.cuda.synchronize()

    _refused(idx, [
        ("search_device short mask", lambda: idx.search_device(q, LENS, K, short_mask)),
        ("search_device short matrix", lambda: idx.search_device(q, LENS, K, short_mat, mask_index_dev=mi)),
        ("search_device float16", lambda: idx.search_device(q16, LENS, K)),
        ("search_device short q", lambda: idx.search_device(q_short, LENS, K)),
        ("search_device out", lambda: idx.search_device(q, LENS, K, out=wide)),
        ("rerank float16", lambda: idx.rerank(q16, LENS, cand, K)),
        ("rerank short q", lambda: idx.rerank(q_short, LENS, cand, K)),
        ("rerank_batch float16", lambda: idx.rerank_batch(q16, LENS, cand2, K)),
        ("rerank_batch short q", lambda: idx.rerank_batch(q_short, LENS, cand2, K)),
        ("rerank_batch out", lambda: idx.rerank_batch(q, LENS, cand2, K, out=wide)),
        ("search_docs_device short mask", lambda: idx.search_docs_device(q, LENS, K, 2, page_doc, N_PAGES, short_mask)),
        ("search_docs_device short matrix",
         lambda: idx.search_docs_device(q, LENS, K, 2, page_doc, N_PAGES, short_mat, mask_index_dev=mi)),
        ("search_docs_device float16", lambda: idx.search_docs_device(q16, LENS, K, 2, page_doc, N_PAGES)),
        ("search_docs_device short q", lambda: idx.search_docs_device(q_short, LENS, K, 2, page_doc, N_PAGES)),
        ("rerank_docs_batch float16", lambda: idx.rerank_docs_batch(q16, LENS, cand2, K, 2, page_doc, N_PAGES)),
        ("rerank_docs_batch short q", lambda: idx.rerank_docs_batch(q_short, LENS, cand2, K, 2, page_doc, N_PAGES)),
        ("sharded_search_begin short matrix", lambda: idx.sharded_search_begin(q, LENS, K, 0, out, short_mat, mi)),
        ("sharded_search_begin float16", lambda: idx.sharded_search_begin(q16, LENS, K, 0, out)),
        ("sharded_search_begin short q", lambda: idx.sharded_search_begin(q_short, LENS, K, 0, out)),
        ("sharded_search_begin out", lambda: idx.sharded_search_begin(q, LENS, K, 0, wide)),
        ("allgather_topk out", lambda: idx.allgather_topk(torch.empty(1024, dtype=torch.uint8, device=dev), n_q, K, out=wide)),
    ])
    idx.close()


def test_two_stage_entry_points_refuse_a_short_mask():
    rng = np.random.default_rng(4)
    two = TwoStageIndex(dtype="bf16")
    two.add_pages(_pages(rng))
    dev = two.device
    queries = [rng.standard_normal((n, 128)).astype(np.float32) for n in LENS]
    mask, short_mask = torch.full((3,), -1, dtype=torch.int32, device=dev), torch.full((2,), -1, dtype=torch.int32, device=dev)
    two.candidates(queries, 10, mask)
    two.search_device(queries, K, 10, mask)
    torch.cuda.synchronize()
    _refused(two.index, [
        ("candidates short mask", lambda: two.candidates(queries, 10, short_mask)),
        ("search_device short mask", lambda: two.search_device(queries, K, 10, short_mask)),
        ("search_device mask matrix", lambda: two.search_device(queries, K, 10, mask.view(1, 3))),
    ])
