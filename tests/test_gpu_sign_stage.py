"""The asymmetric sign stage on the GPU (run with -m gpu on an H100): b200ms_sign_rows / b200ms_set_sign_rows /
b200ms_sign_candidates_device and signs.SignTwoStageIndex, over bf16, int8 and fp8 planted corpora (oracle/planted.py: empty
pages, partial chunks, pages longer than a work unit) in HBM and in pinned host memory.

  * sign rows equal b200ms_sign_pack of the widened packed rows, bit for bit, padding rows included;
  * candidate scores are tests/sign_oracle.py's exact integers and ids follow its order, for query lengths 0 / 1 / 31 / 32 /
    33 / 64 and batches of 1 / 2 / 4 / 8 / 9 / 64 queries (every resident-tile count and the split launch);
  * masks (one for all, per query, index -1), with the filtered scan plan forced and not, and n_cand 1 / all / 4096;
  * the two-stage result is rerank_batch over the candidate list, and the exhaustive search when every page is a candidate;
  * the host tier equals the HBM tier bit for bit;
  * append, compaction and save / load / open keep the sign rows equal to a fresh rebuild;
  * refused calls launch nothing;
  * cross-stream ordering: a sign-candidate call in flight on one stream while the next call of the handle runs on another
    (these exports name their stream `cuda_stream`, so their cases live here rather than in tests/stream_order_cases.py);
  * the store: query_similar / query_similar_documents with doc_ids in sign-candidate mode return the exhaustive winners.
"""
import asyncio
import ctypes

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

torch = pytest.importorskip("torch")
if not torch.cuda.is_available():  # pragma: no cover - the gpu marker normally deselects these on CPU boxes
    pytest.skip("CUDA device required", allow_module_level=True)

import sign_oracle as so  # noqa: E402
from morphik_core_b200 import _native as nat  # noqa: E402
from morphik_core_b200.index import _aligned_bytes  # noqa: E402
from morphik_core_b200.models import DocumentChunk  # noqa: E402
from morphik_core_b200.signs import SignTwoStageIndex  # noqa: E402
from morphik_core_b200.store import B200MultiVectorStore  # noqa: E402
from oracle.planted import planted_corpus, planted_queries  # noqa: E402

DEV = torch.device("cuda", 0)
DTYPES = ("bf16", "int8", "fp8")
LENS = (0, 1, 31, 32, 33, 64)
Q_SCALE = 127.0


def cstream(s=None):
    return ctypes.c_void_p((s or torch.cuda.current_stream(DEV)).cuda_stream)


@pytest.fixture(scope="module", params=[(d, t) for d in DTYPES for t in ("hbm", "host")], ids=lambda p: f"{p[0]}-{p[1]}")
def built(request):
    dtype, tier = request.param
    pc = planted_corpus(dtype, seed=3)
    sti = SignTwoStageIndex(dtype=dtype, tier=tier, q_scale=Q_SCALE)
    sti.add_pages(pc.pages)
    torch.cuda.synchronize(DEV)
    packed = sti.index.packed_rows().cpu().numpy()
    bits = so.sign_bits(dtype, packed)
    yield dtype, tier, pc, sti, bits
    torch.cuda.synchronize(DEV)
    sti.index.close()


def queries_for(pc, n_q, seed=1):
    return planted_queries(pc, [LENS[i % len(LENS)] for i in range(n_q)], seed=seed)


def raw_candidates(sti, queries, n_cand, masks=None, index=None, stream=None):
    """b200ms_sign_candidates_device with score_scale 1 (scores are the exact integers S), on `stream`."""
    src, _ = sti.index._stage_rows(list(queries))
    lens = [int(q.shape[0]) for q in queries]
    n_q = len(lens)
    ts = torch.empty((n_q, n_cand), dtype=torch.float32, device=DEV)
    ti = torch.empty((n_q, n_cand), dtype=torch.int64, device=DEV)
    tc = torch.empty((n_q,), dtype=torch.int32, device=DEV)
    sti._attach()
    rc = nat.lib.b200ms_sign_candidates_device(
        sti.index.h.ptr, ctypes.c_void_p(src.data_ptr()), nat.F32 if src.dtype == torch.float32 else nat.BF16,
        nat.i32_array(lens), n_q, n_cand, None if masks is None else ctypes.c_void_p(masks.data_ptr()),
        0 if masks is None else masks.shape[0], None if index is None else ctypes.c_void_p(index.data_ptr()),
        ctypes.c_float(Q_SCALE), ctypes.c_float(1.0), ctypes.c_void_p(ts.data_ptr()), ctypes.c_void_p(ti.data_ptr()),
        ctypes.c_void_p(tc.data_ptr()), cstream(stream))
    sti.index.h.check(rc, "b200ms_sign_candidates_device")
    return ts, ti, tc


def oracle_scores(queries, bits, pc):
    return so.scores([so.quantise_query(q, Q_SCALE) for q in queries], bits, pc.lens)


def check_candidates(res, S, n_cand, allowed_rows):
    ts, ti, tc = (t.cpu().numpy() for t in res)
    for q in range(S.shape[0]):
        want = so.topk(S[q], n_cand, allowed_rows[q])
        assert tc[q] == len(want), q
        assert ti[q, :len(want)].tolist() == want, q
        np.testing.assert_array_equal(ts[q, :len(want)], S[q, want].astype(np.float32))
        assert (ti[q, len(want):] == -1).all() and np.isneginf(ts[q, len(want):]).all()


def test_sign_rows_equal_sign_pack_of_the_widened_rows(built):
    dtype, _, pc, sti, bits = built
    packed = torch.from_numpy(sti.index.packed_rows().cpu().numpy()).to(DEV)
    if dtype == "bf16":
        wide = packed.view(torch.bfloat16).float()
    elif dtype == "int8":
        wide = packed.view(torch.int8).float()
    else:
        wide = packed.view(torch.float8_e4m3fn).float()
    want = sti.index.sign_pack(wide.view(-1, 128).contiguous()).cpu().numpy()
    got = sti.sign_rows().cpu().numpy()
    assert got.shape == (sti.index.n_rows_padded, 16)
    np.testing.assert_array_equal(got, want)
    np.testing.assert_array_equal(got, so.pack_bits(bits))


@pytest.mark.parametrize("n_q", [1, 2, 4, 8, 9, 64])
def test_scores_are_the_oracle_integers(built, n_q):
    _, _, pc, sti, bits = built
    qs = queries_for(pc, n_q, seed=n_q)
    S = oracle_scores(qs, bits, pc)
    res = raw_candidates(sti, qs, 4096)
    check_candidates(res, S, 4096, [None] * n_q)


@pytest.mark.parametrize("max_ctas", [0, 8])  # 8: more work units than CTAs, so masked calls walk the filtered plan
def test_masks_match_the_masked_oracle_topk(built, max_ctas):
    _, _, pc, sti, bits = built
    n = sti.n_pages
    words = (n + 31) // 32
    rng = np.random.default_rng(7)
    sti.index.set_option("max_ctas", max_ctas)
    try:
        qs = queries_for(pc, 9, seed=11)
        S = oracle_scores(qs, bits, pc)
        mats = rng.integers(0, 2**32, size=(3, words), dtype=np.uint64).astype(np.uint32)
        mats[2] = 0
        mats[2, 0] = 0b1010  # two pages
        allow = [so.mask_allowed(m, n) for m in mats]
        index = np.array([0, 1, -1, 2, 0, 1, 2, -1, 0], dtype=np.int32)
        rows = [None if i < 0 else allow[i] for i in index]
        masks_dev = torch.from_numpy(mats.view(np.int32)).to(DEV)
        index_dev = torch.from_numpy(index).to(DEV)
        n_allowed = int(max(a.sum() for a in allow))
        for n_cand in (1, n_allowed, 4096):
            check_candidates(raw_candidates(sti, qs, n_cand, masks_dev, index_dev), S, n_cand, rows)
        one = masks_dev[1:2].contiguous()  # one mask for every query
        check_candidates(raw_candidates(sti, qs, 5, one, torch.zeros(9, dtype=torch.int32, device=DEV)), S, 5, [allow[1]] * 9)
    finally:
        sti.index.set_option("max_ctas", 0)


def test_two_stage_is_the_rerank_of_the_candidates(built):
    dtype, tier, pc, sti, _ = built
    qs = planted_queries(pc, [1, 31, 32, 33, 64], seed=5)
    lens = [int(q.shape[0]) for q in qs]
    src, _ = sti.index._stage_rows(qs)
    for n_cand in (3, 4096):
        _, ci, _ = sti.candidates_device(src, lens, sti._n_cand(max(n_cand, 10)))  # search_device's candidate count
        want = sti.index.rerank_batch(src, lens, ci, 10)
        got = sti.search_device(qs, 10, n_candidates=n_cand)[:3]
        for a, b in zip(got, want):
            assert torch.equal(a, b)
    if tier == "hbm":  # every page a candidate: the exhaustive search, bit for bit
        full = sti.index.search_device(src, lens, 10)
        got = sti.search_device(qs, 10, n_candidates=4096)[:3]
        for a, b in zip(got, full):
            assert torch.equal(a, b)


def test_host_tier_equals_hbm_tier():
    for dtype in DTYPES:
        pc = planted_corpus(dtype, seed=3)
        a, b = SignTwoStageIndex(dtype=dtype, tier="hbm"), SignTwoStageIndex(dtype=dtype, tier="host")
        a.add_pages(pc.pages)
        b.add_pages(pc.pages)
        qs = queries_for(pc, 9, seed=2)
        assert torch.equal(a.sign_rows(), b.sign_rows())
        for x, y in zip(a.candidates(qs, 50), b.candidates(qs, 50)):
            assert torch.equal(x, y)
        for x, y in zip(a.search(qs, 10, 40), b.search(qs, 10, 40)):
            np.testing.assert_array_equal(x, y)
        a.index.close()
        b.index.close()


@pytest.mark.parametrize("tier", ["hbm", "host"])
def test_append_and_compact_keep_the_signs_of_a_rebuild(tier):
    pc = planted_corpus("bf16", seed=4)
    sti = SignTwoStageIndex(dtype="bf16", tier=tier)
    third = len(pc.pages) // 3
    for part in (pc.pages[:third], pc.pages[third:2 * third], pc.pages[2 * third:]):
        sti.add_pages(part)
    grown = sti.sign_rows().clone()
    sti.rebuild_from_index()
    assert torch.equal(grown, sti.sign_rows())
    keep = [p for p in range(sti.n_pages) if p % 3 != 1]
    sti.compact(keep)
    compacted = sti.sign_rows().clone()
    sti.rebuild_from_index()
    assert torch.equal(compacted, sti.sign_rows())
    fresh = SignTwoStageIndex(dtype="bf16", tier=tier)
    fresh.add_pages([pc.pages[p] for p in keep])
    assert torch.equal(compacted, fresh.sign_rows())
    qs = queries_for(pc, 4, seed=9)
    for x, y in zip(sti.search(qs, 5, 30), fresh.search(qs, 5, 30)):
        np.testing.assert_array_equal(x, y)
    sti.index.close()
    fresh.index.close()


def test_refused_calls_launch_nothing():
    h = nat.Handle(0)
    q = torch.zeros((4, 128), dtype=torch.float32, device=DEV)
    out = [torch.empty(64, dtype=dt, device=DEV) for dt in (torch.float32, torch.int64, torch.int32)]
    lens = nat.i32_array([4])

    def cands(n_cand=4, scale=1.0, lens_=lens, n_q=1):
        return nat.lib.b200ms_sign_candidates_device(h.ptr, ctypes.c_void_p(q.data_ptr()), nat.F32, lens_, n_q, n_cand, None, 0,
                                                     None, ctypes.c_float(scale), ctypes.c_float(1.0),
                                                     *[ctypes.c_void_p(t.data_ptr()) for t in out], cstream())

    before = nat.lib.b200ms_launch_count(h.ptr)
    assert cands() == -3  # B200MS_ESTATE: no corpus
    sign_buf = _aligned_bytes(64 * 16, DEV, 16)
    assert nat.lib.b200ms_sign_rows(h.ptr, 0, 1, ctypes.c_void_p(sign_buf.data_ptr()), cstream()) == -3
    rows = _aligned_bytes(96 * 256, DEV)  # pages of 40, 0 and 3 rows: 64 + 32 padded rows
    page_lens = nat.i32_array([40, 0, 3])
    h.check(nat.lib.b200ms_set_corpus(h.ptr, ctypes.c_void_p(rows.data_ptr()), nat.BF16, page_lens, 3))
    before = nat.lib.b200ms_launch_count(h.ptr)
    assert cands() == -3  # no sign rows attached
    assert nat.lib.b200ms_set_sign_rows(h.ptr, ctypes.c_void_p(sign_buf.data_ptr()), 63, cstream()) == -1  # 96 rows
    assert nat.lib.b200ms_set_sign_rows(h.ptr, ctypes.c_void_p(sign_buf.data_ptr() + 8), 96, cstream()) == -1
    assert nat.lib.b200ms_sign_rows(h.ptr, 2, 2, ctypes.c_void_p(sign_buf.data_ptr()), cstream()) == -1
    signs = _aligned_bytes(96 * 16, DEV, 16)
    h.check(nat.lib.b200ms_set_sign_rows(h.ptr, ctypes.c_void_p(signs.data_ptr()), 96, cstream()))
    for kw in ({"n_cand": 0}, {"n_cand": 4097}, {"scale": 0.0}, {"scale": -1.0}, {"scale": float("inf")},
               {"scale": float("nan")}, {"n_q": 0}, {"lens_": nat.i32_array([-1])}):
        assert cands(**kw) == -1, kw
    assert nat.lib.b200ms_launch_count(h.ptr) == before
    assert cands() == 0 and nat.lib.b200ms_launch_count(h.ptr) > before
    # set_corpus detaches the signs
    h.check(nat.lib.b200ms_set_corpus(h.ptr, ctypes.c_void_p(rows.data_ptr()), nat.BF16, page_lens, 3))
    before = nat.lib.b200ms_launch_count(h.ptr)
    assert cands() == -3
    b1 = _aligned_bytes(96 * 16, DEV)
    h.check(nat.lib.b200ms_set_corpus(h.ptr, ctypes.c_void_p(b1.data_ptr()), nat.B1, page_lens, 3))
    before = nat.lib.b200ms_launch_count(h.ptr)
    assert nat.lib.b200ms_sign_rows(h.ptr, 0, 1, ctypes.c_void_p(sign_buf.data_ptr()), cstream()) == -3
    assert nat.lib.b200ms_set_sign_rows(h.ptr, ctypes.c_void_p(b1.data_ptr()), 96, cstream()) == -3
    assert nat.lib.b200ms_launch_count(h.ptr) == before
    torch.cuda.synchronize(DEV)
    h.close()


def test_cross_stream_order():
    """Call A (a 64-query sign-candidate scan) in flight on stream 1; call B of the same handle on stream 2 at once:
    b200ms_sign_rows into a fresh buffer, b200ms_set_sign_rows, another sign-candidate call.  Each result equals its solo
    run bit for bit."""
    pc = planted_corpus("int8", seed=6)
    sti = SignTwoStageIndex(dtype="int8")
    sti.add_pages(pc.pages * 6)
    qa = queries_for(pc, 64, seed=1)
    qb = queries_for(pc, 3, seed=2)
    solo_a = [t.clone() for t in raw_candidates(sti, qa, 500)]
    solo_b = [t.clone() for t in raw_candidates(sti, qb, 20)]
    solo_rows = sti.sign_rows().clone()
    torch.cuda.synchronize(DEV)
    s1, s2 = torch.cuda.Stream(DEV), torch.cuda.Stream(DEV)
    fresh = _aligned_bytes(sti.index.n_rows_padded * 16, DEV, 16)
    fresh.zero_()
    torch.cuda.synchronize(DEV)
    with torch.cuda.stream(s1):
        got_a = raw_candidates(sti, qa, 500, stream=s1)
    with torch.cuda.stream(s2):
        sti.index.h.check(nat.lib.b200ms_sign_rows(sti.index.h.ptr, 0, sti.n_pages, ctypes.c_void_p(fresh.data_ptr()),
                                                   cstream(s2)))
        sti.index.h.check(nat.lib.b200ms_set_sign_rows(sti.index.h.ptr, ctypes.c_void_p(fresh.data_ptr()),
                                                       sti.index.n_rows_padded, cstream(s2)))
        got_b = raw_candidates(sti, qb, 20, stream=s2)
    torch.cuda.synchronize(DEV)
    for x, y in zip(got_a, solo_a):
        assert torch.equal(x, y)
    for x, y in zip(got_b, solo_b):
        assert torch.equal(x, y)
    assert torch.equal(fresh.view(-1, 16), solo_rows)
    sti.index.close()


def _run(coro):
    return asyncio.run(coro)


def test_store_routes_through_signs_and_persists(tmp_path):
    pc = planted_corpus("bf16", seed=8)
    chunks = [DocumentChunk(document_id=f"d{i % 5}", chunk_number=i, content=str(i), embedding=p, metadata={})
              for i, p in enumerate(pc.pages) if len(p)]
    ex = B200MultiVectorStore(mode="bf16")
    st = B200MultiVectorStore(mode="bf16", sign_candidates=4096)  # every allowed page is a candidate: exhaustive results
    for s in (ex, st):
        _run(s.store_embeddings(chunks))
    q = planted_queries(pc, [33], seed=4)[0]
    for doc_ids in (None, ["d1", "d3"]):
        a = _run(ex.query_similar(q, k=6, doc_ids=doc_ids))
        b = _run(st.query_similar(q, k=6, doc_ids=doc_ids))
        assert [(r.document_id, r.chunk_number, r.score) for r in a] == [(r.document_id, r.chunk_number, r.score) for r in b]
        a = _run(ex.query_similar_documents(q, k=2, pages_per_document=2, doc_ids=doc_ids))
        b = _run(st.query_similar_documents(q, k=2, pages_per_document=2, doc_ids=doc_ids))
        assert [[(r.chunk_number, r.score) for r in d] for d in a] == [[(r.chunk_number, r.score) for r in d] for d in b]
    assert "sign_candidates_ms" in _run(_timed(st, q))
    st.save(str(tmp_path / "saved"))
    loaded = B200MultiVectorStore.load(str(tmp_path / "saved"), sign_candidates=4096)
    assert torch.equal(loaded._two_stage.sign_rows(), st._two_stage.sign_rows())
    jd = str(tmp_path / "journal")
    op = B200MultiVectorStore.open(jd, mode="bf16", sign_candidates=4096)
    _run(op.store_embeddings(chunks[:10]))
    _run(op.store_embeddings(chunks[10:]))
    op.close()
    reopened = B200MultiVectorStore.open(jd, mode="bf16", sign_candidates=4096)
    assert torch.equal(reopened._two_stage.sign_rows(), st._two_stage.sign_rows())
    r1 = _run(reopened.query_similar(q, k=6, doc_ids=["d2"]))
    r2 = _run(ex.query_similar(q, k=6, doc_ids=["d2"]))
    assert [(r.chunk_number, r.score) for r in r1] == [(r.chunk_number, r.score) for r in r2]
    for s in (ex, st, loaded, reopened):
        s.close()


async def _timed(store, q):
    await store.query_similar_batch([q], k=3)
    return store.last_query_timing
