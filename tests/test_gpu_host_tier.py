"""Host-resident corpora (run with -m gpu on an H100): packed rows in pinned host memory, rerank candidates gathered over PCIe.

The host tier must be indistinguishable from the HBM tier on the same packed rows and candidate lists: scores, ids, counts
and tie order bit for bit, for every corpus dtype, shared and per-query lists (duplicates within and across queries, -1 and
ids past the corpus), zero_pad_compat, several staging rounds, and through the FDE, two-stage and store layers.  Pinned
allocations stay far below 1 GB.
"""
import asyncio
import ctypes
import functools

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

torch = pytest.importorskip("torch")
if not torch.cuda.is_available():  # pragma: no cover - the gpu marker normally deselects these on CPU boxes
    pytest.skip("CUDA device required", allow_module_level=True)

from morphik_core_b200 import _native as nat  # noqa: E402
from morphik_core_b200.fde import TwoStageIndex  # noqa: E402
from morphik_core_b200.index import MaxSimIndex  # noqa: E402
from morphik_core_b200.models import DocumentChunk  # noqa: E402
from morphik_core_b200.store import B200MultiVectorStore  # noqa: E402
from oracle import planted  # noqa: E402
from oracle.scoring import assert_candidate_ranking, oracle_scores, slot_scores_of  # noqa: E402

DTYPES = ["bf16", "int8", "fp8", "binary"]
RERANK_T = [5, 17, 32, 9, 1, 33, 130, 300]  # queries of 1 .. 300 tokens, four 1-group queries sharing a tile


@functools.lru_cache(maxsize=None)
def corpus(dtype):
    return planted.planted_corpus(dtype, seed=2024, n_random=40)


@functools.lru_cache(maxsize=None)
def queries(dtype):
    return planted.planted_queries(corpus(dtype), RERANK_T, seed=6)


def pair(dtype, pages, zero_pad=0):
    """HBM-tier and host-tier indexes over the same pages."""
    out = []
    for tier in ("hbm", "host"):
        idx = MaxSimIndex(dtype=dtype, tier=tier)
        if zero_pad:
            idx.set_option("zero_pad_compat", zero_pad)
        idx.add_pages(pages)
        out.append(idx)
    hbm, host = out
    assert host.packed_rows().device.type == "cpu"
    assert torch.equal(hbm.packed_rows().cpu(), host.packed_rows())
    return hbm, host


def rerank(idx, qs, cand, k):
    qd = torch.from_numpy(np.concatenate(qs).astype(np.float32)).cuda()
    cd = torch.from_numpy(np.ascontiguousarray(cand, np.int64)).cuda()
    lens = [len(q) for q in qs]
    ts, ti, tc = idx.rerank_batch(qd, lens, cd, k) if cd.ndim == 2 else idx.rerank(qd, lens, cd, k)
    torch.cuda.synchronize()
    return ts.cpu().numpy(), ti.cpu().numpy(), tc.cpu().numpy()


def assert_identical(a, b, what):
    for x, y, name in zip(a, b, ("scores", "ids", "counts")):
        assert x.shape == y.shape and np.array_equal(x.view(np.uint8), y.view(np.uint8)), (what, name)


def candidate_lists(rng, n_pages, n_lists, n_cand, empty_pages):
    """Random lists with duplicates within a list, -1 slots, ids past the corpus and empty pages; lists drawn from one
    corpus overlap, so pages repeat across queries too."""
    cand = np.stack([rng.permutation(n_pages)[:n_cand] for _ in range(n_lists)]).astype(np.int64)
    for i in range(n_lists):
        cand[i, 3] = cand[i, 1]
        cand[i, n_cand - 1] = cand[i, 0]
        cand[i, 5] = -1
        cand[i, 8] = n_pages
        cand[i, 9 + i % 5] = n_pages + 1000 * i + 7
        cand[i, 20] = empty_pages[i % len(empty_pages)]
        if i:
            cand[i, 30] = cand[i - 1, 31]  # the same page in two queries' lists
    return cand


def expected_traffic(idx, cand):
    """(unique valid pages, padded bytes) of a call's candidate slots, counted in numpy."""
    c = np.asarray(cand).reshape(-1)
    u = np.unique(c[(c >= 0) & (c < idx.n_pages)])
    pad = (idx.page_lens[u].astype(np.int64) + 31) // 32 * 32
    return len(u), int(pad.sum()) * idx.row_bytes


@pytest.mark.parametrize("dtype", DTYPES)
def test_host_tier_rerank_identical_to_hbm_and_oracle(dtype):
    pc = corpus(dtype)
    hbm, host = pair(dtype, pc.pages)
    n_pages = len(pc.pages)
    empty = [p for p, n in enumerate(pc.lens) if n == 0]
    qs = queries(dtype)
    want = oracle_scores(dtype, qs, pc.pages)
    rng = np.random.default_rng(8)
    n_cand = 48
    per_q = candidate_lists(rng, n_pages, len(qs), n_cand, empty)
    shared = candidate_lists(rng, n_pages, 1, n_cand, empty)[0]
    for k in (7, n_cand):
        for cand in (per_q, shared):
            what = f"{dtype} k={k} {'per-query' if cand.ndim == 2 else 'shared'}"
            got = rerank(host, qs, cand, k)
            assert_identical(got, rerank(hbm, qs, cand, k), what)
            st = host.gather_stats()
            assert (st["unique_pages"], st["bytes"]) == expected_traffic(host, cand), (what, st)
            assert st["rounds"] == 1 and st["ms"] >= 0.0
            for qi in range(len(qs)):
                c = cand[qi] if cand.ndim == 2 else cand
                assert_candidate_ranking(dtype, got[0][qi], got[1][qi], got[2][qi], slot_scores_of(want[qi], c), c, n_pages, k,
                                         f"{what} q{qi}")


@pytest.mark.parametrize("dtype", DTYPES)
def test_staging_rounds_identical_to_one_round(dtype):
    pc = corpus(dtype)
    hbm, host = pair(dtype, pc.pages)
    qs = queries(dtype)
    rng = np.random.default_rng(11)
    cand = candidate_lists(rng, len(pc.pages), len(qs), 64, [p for p, n in enumerate(pc.lens) if n == 0])
    one = rerank(host, qs, cand, 20)
    assert host.gather_stats()["rounds"] == 1
    _, nbytes = expected_traffic(host, cand)
    host.set_option("host_stage_bytes", max(nbytes // 4, 1))  # raised to the largest page if smaller
    for c in (cand, cand[0]):
        many = rerank(host, qs, c, 20)
        st = host.gather_stats()
        assert st["rounds"] >= 3, st
        assert (st["unique_pages"], st["bytes"]) == expected_traffic(host, c)
        assert_identical(many, rerank(hbm, qs, c, 20), f"{dtype} rounds={st['rounds']}")
    assert_identical(rerank(host, qs, cand, 20), one, f"{dtype} rounds vs one round")
    host.set_option("host_stage_bytes", 1)  # every round holds about one page
    assert_identical(rerank(host, qs, cand, 20), one, f"{dtype} one page per round")


@pytest.mark.parametrize("batch", [3, 128])
@pytest.mark.parametrize("dtype", ["bf16", "int8", "fp8"])
def test_zero_pad_compat_identical(dtype, batch):
    rng = np.random.default_rng(29 + batch)
    lens = [int(x) for x in rng.integers(1, 200, size=150)] + [0, 400, 3]
    pages = [np.abs(rng.standard_normal((n, 128))).astype(np.float32) / 12 for n in lens]
    qs = [(rng.standard_normal((t, 128)) / 12 - (0.3 if i % 2 else 0)).astype(np.float32) for i, t in enumerate([3, 40, 130])]
    hbm, host = pair(dtype, pages, zero_pad=batch)
    cand = np.stack([rng.permutation(len(lens))[:140] for _ in qs]).astype(np.int64)
    cand[:, 7] = -1
    for c in (cand, cand[1]):
        assert_identical(rerank(host, qs, c, 50), rerank(hbm, qs, c, 50), f"{dtype} zero_pad={batch}")


@pytest.mark.parametrize("dtype", DTYPES)
def test_single_page_corpus_and_all_slots_invalid(dtype):
    rng = np.random.default_rng(5)
    hbm, host = pair(dtype, [(rng.standard_normal((37, 128)) / 11).astype(np.float32)])
    qs = [(rng.standard_normal((t, 128)) / 11).astype(np.float32) for t in (1, 33)]
    for cand in (np.array([0, -1, 0, 5], np.int64), np.array([[0, 0, -1], [-1, 3, 0]], np.int64),
                 np.array([-1, 7, -1], np.int64), np.array([[-1, 1], [9, -1]], np.int64)):
        got = rerank(host, qs, cand, 3)
        assert_identical(got, rerank(hbm, qs, cand, 3), f"{dtype} {cand.tolist()}")
        assert host.gather_stats()["unique_pages"] == expected_traffic(host, cand)[0]
    assert np.all(got[2] == 0) and host.gather_stats()["rounds"] == 0


def test_full_scans_refused_and_bad_memory_rejected():
    rng = np.random.default_rng(1)
    host = MaxSimIndex(dtype="bf16", tier="host")
    host.add_pages([(rng.standard_normal((40, 128)) / 11).astype(np.float32) for _ in range(3)])
    q = [(rng.standard_normal((8, 128)) / 11).astype(np.float32)]
    qd = torch.from_numpy(q[0]).cuda()
    for call in (lambda: host.search_host(q, 2), lambda: host.search_host_masked(q, 2, [None]),
                 lambda: host.search_device(qd, [8], 2), lambda: host.score_matrix(q)):
        with pytest.raises(nat.NativeError, match="only candidate scoring"):
            call()
    lens = nat.i32_array([40])
    dev = torch.zeros(1 << 14, dtype=torch.uint8, device="cuda")
    pageable = np.zeros(1 << 14, dtype=np.uint8)
    h = host.h
    assert nat.lib.b200ms_set_corpus_host(h.ptr, ctypes.c_void_p(dev.data_ptr()), nat.BF16, lens, 1) == nat_einval()
    assert nat.lib.b200ms_set_corpus_host(h.ptr, pageable.ctypes.data_as(ctypes.c_void_p), nat.BF16, lens, 1) == nat_einval()
    assert "pinned" in nat.lib.b200ms_last_error(h.ptr).decode()
    blk = host._block.ptr
    assert nat.lib.b200ms_set_corpus_host(h.ptr, ctypes.c_void_p(blk + 8), nat.BF16, lens, 1) == nat_einval()  # alignment
    host._attached = False  # the refused calls above left the old corpus attached; re-attach for the checks below
    ts, ti, tc = host.rerank(qd, [8], torch.tensor([2, 0], dtype=torch.int64, device="cuda"), 2)
    assert int(tc[0]) == 2


def nat_einval():
    return -1


def test_fde_encode_corpus_identical_through_the_mapping():
    rng = np.random.default_rng(4)
    lens = [int(x) for x in rng.integers(1, 300, size=70)] + [0, 1030, 32]
    pages = [(rng.standard_normal((n, 128)) / 11).astype(np.float32) for n in lens]
    a, b = TwoStageIndex(dtype="bf16"), TwoStageIndex(dtype="bf16", tier="host")
    a.add_pages(pages)
    b.add_pages(pages)
    a.rebuild_from_index(batch_pages=16)
    b.rebuild_from_index(batch_pages=16)
    fa, ia = a.fde_rows()
    fb, ib = b.fde_rows()
    assert torch.equal(fa.view(torch.int16), fb.view(torch.int16)) and torch.equal(ia.view(torch.int32), ib.view(torch.int32))
    qs = [(rng.standard_normal((t, 128)) / 11).astype(np.float32) for t in (32, 7, 64)]
    sa = a.search(qs, k=10, n_candidates=30)
    sb = b.search(qs, k=10, n_candidates=30)
    assert_identical(sa, sb, "two-stage host vs hbm")
    t = b.last_timing_ms
    assert t["gather_pages"] > 0 and t["gather_bytes"] > 0 and t["load_multivectors_ms"] > 0.0
    assert a.last_timing_ms["load_multivectors_ms"] == 0.0


def test_hbm_footprint_of_host_tier():
    rng = np.random.default_rng(2)
    pages = [(rng.standard_normal((1024, 128)) / 11).astype(np.float32) for _ in range(256)]  # 64 MB of bf16 rows
    idx = MaxSimIndex(dtype="bf16", tier="host")
    idx.add_pages(pages[:8])
    torch.cuda.synchronize()
    before = torch.cuda.memory_allocated()
    for i in range(8, 256, 32):
        idx.add_pages(pages[i:i + 32])
    torch.cuda.synchronize()
    grown = torch.cuda.memory_allocated() - before
    assert grown < 0.1 * 248 * 1024 * 256, grown
    assert idx.packed_rows().device.type == "cpu" and idx.n_rows_padded == 256 * 1024


def _run(coro):
    return asyncio.run(coro)


def _chunks(rng, n_docs, per_doc, base=0):
    out = []
    for d in range(n_docs):
        for j in range(per_doc):
            n = int(rng.integers(1, 200))
            out.append(DocumentChunk(document_id=f"d{base + d}", content=f"d{base + d}/{j}", chunk_number=j, metadata={},
                                     embedding=(rng.standard_normal((n, 128)) / 11).astype(np.float32)))
    return out


def _results(store, qs, k=8):
    res = []
    for q in qs:
        got = _run(store.query_similar(q, k))
        res.append([(c.document_id, c.chunk_number, np.float32(c.score).tobytes()) for c in got])
    return res


def test_store_host_tier_identical_to_hbm(tmp_path):
    rng = np.random.default_rng(12)
    chunks = _chunks(rng, 12, 4)
    qs = [(rng.standard_normal((t, 128)) / 11).astype(np.float32) for t in (20, 33, 5)]
    kw = dict(fde_candidates=24, compact_dead_fraction=0.05)
    a = B200MultiVectorStore(**kw)
    b = B200MultiVectorStore(corpus_tier="host", **kw)
    assert b._index.tier == "host"
    for s in (a, b):
        _run(s.store_embeddings(chunks[:30]))
        _run(s.store_embeddings(chunks[30:]))
    assert _results(a, qs) == _results(b, qs)
    for s in (a, b):
        assert _run(s.delete_chunks_by_document_id("d3"))  # past the dead fraction: compacts
    assert b._index.n_pages == len(chunks) - 4
    assert _results(a, qs) == _results(b, qs)
    a.save(str(tmp_path / "a"))
    b.save(str(tmp_path / "b"))
    la = B200MultiVectorStore.load(str(tmp_path / "a"), fde_candidates=24)
    lb = B200MultiVectorStore.load(str(tmp_path / "b"), fde_candidates=24, corpus_tier="host")
    assert lb._index.tier == "host"
    assert _results(la, qs) == _results(a, qs) == _results(lb, qs)
    # journal replay: segments read straight into the host block
    ja = B200MultiVectorStore.open(str(tmp_path / "ja"), **kw)
    jb = B200MultiVectorStore.open(str(tmp_path / "jb"), corpus_tier="host", **kw)
    more = _chunks(rng, 3, 2, base=50)
    for s in (ja, jb):
        _run(s.store_embeddings(chunks[:20]))
        _run(s.store_embeddings(more))
        _run(s.delete_chunks_by_document_id("d1"))
    ra = B200MultiVectorStore.open(str(tmp_path / "ja"), **kw)
    rb = B200MultiVectorStore.open(str(tmp_path / "jb"), corpus_tier="host", **kw)
    assert rb._index.tier == "host"
    assert _results(ra, qs) == _results(ja, qs) == _results(jb, qs) == _results(rb, qs)
