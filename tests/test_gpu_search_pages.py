"""Searching with stored pages as the queries on an H100 (run with -m gpu): b200ms_search_pages_device,
b200ms_rerank_pages_batch_device and b200ms_page_rows_device through MaxSimIndex, the two first stages and the store.

- identity: for bf16, fp8 and binary corpora, search_pages([p, ...]) returns search_device's ids, counts and tie order for
  the pages' dequantised rows as float queries, with scores bit for bit search_device's over the source's row count, with
  and without per-source masks;
- int8 is exact: integer MaxSim over the codes in int64 through the I32 sum rule, a 1100-row +-127 / -128 source included;
- bf16 against the float64 page-to-page MaxSim of tests/mmr_oracle.py at page lengths 0, 1, 31, 33, 1024 and 1500;
- the host tier reranks bit-identically to HBM and gathers only the candidate pages; FDE and sign two-stage searches with
  every page as a candidate equal the exhaustive search;
- refusals launch nothing; a call in flight on another stream of the same handle.
"""
import asyncio
import ctypes

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

torch = pytest.importorskip("torch")
if not torch.cuda.is_available():  # pragma: no cover - the gpu marker normally deselects these on CPU boxes
    pytest.skip("CUDA device required", allow_module_level=True)

from mmr_oracle import page_sum  # noqa: E402
from morphik_core_b200 import _native as nat  # noqa: E402
from morphik_core_b200.index import MaxSimIndex  # noqa: E402
from morphik_core_b200.models import DocumentChunk  # noqa: E402
from morphik_core_b200.store import B200MultiVectorStore  # noqa: E402
from oracle import maxsim_oracle as orc  # noqa: E402
from oracle.scoring import TOL, i32_reported, i32_sum  # noqa: E402

DEV = torch.device("cuda", 0)
LENS = [0, 1, 31, 32, 33, 64, 65, 200, 1024, 1500, 17, 90, 3, 128, 40]


def _unit(rng, n):
    x = rng.standard_normal((n, 128)).astype(np.float32)
    return x / np.maximum(np.linalg.norm(x, axis=1, keepdims=True), 1e-9)


def _pages(seed=5, lens=LENS):
    rng = np.random.default_rng(seed)
    pages = [_unit(rng, n) for n in lens]
    pages.append(pages[7].copy())  # an exact copy: a tie with the source's own page
    return pages


PAGES = _pages()
_IDX = {}


def _index(dtype, tier="hbm"):
    if (dtype, tier) not in _IDX:
        idx = MaxSimIndex(dtype=dtype, tier=tier)
        idx.add_pages(PAGES)
        idx._attach()
        _IDX[(dtype, tier)] = idx
    return _IDX[(dtype, tier)]


def bits(x):
    return np.ascontiguousarray(x, np.float32).view(np.uint32)


def host(ts):
    return tuple(t.cpu().numpy() for t in ts)


def dequantised(idx, p):
    """Page p's true rows from the packed corpus, as the float values the scan multiplies (the comparison query)."""
    lens = idx.page_lens.astype(np.int64)
    r0 = int(((lens[:p] + 31) // 32 * 32).sum())
    raw = idx.packed_rows()[r0:r0 + int(lens[p])].cpu().numpy()
    if idx.dtype == nat.BF16:
        return (raw.view(np.uint16).astype(np.uint32) << 16).view(np.float32)
    if idx.dtype == nat.F8:
        return orc.dequantize_e4m3_np(raw) / np.float32(idx.i8_scale)
    if idx.dtype == nat.I8:
        return raw.view(np.int8).astype(np.float32) / np.float32(idx.i8_scale)
    return np.where(np.unpackbits(raw, axis=1) > 0, 1.0, -1.0).astype(np.float32)


def reference(idx, src, k, masks=None, index=None):
    """search_device over the sources' dequantised rows: (scores / len in float32, ids, counts)."""
    qs = [dequantised(idx, p) for p in src]
    q = torch.from_numpy(np.concatenate(qs)).to(DEV)
    ts, ti, tc = host(idx.search_device(q, [len(x) for x in qs], k, allow_mask_dev=masks, mask_index_dev=index))
    lens = np.asarray([len(x) for x in qs], np.float32)[:, None]
    return ts / lens, ti, tc


def random_masks(idx, n, seed):
    rng = np.random.default_rng(seed)
    words = [idx.mask_from_pages(rng.random(idx.n_pages) < f) for f in (0.6, 0.3)]
    masks = torch.from_numpy(np.stack(words).view(np.int32)).to(DEV)
    index = torch.tensor([i % 3 - 1 for i in range(n)], dtype=torch.int32, device=DEV)
    return masks, index


@pytest.mark.parametrize("dtype", ["bf16", "fp8", "binary"])
def test_identity_with_search_device(dtype):
    idx = _index(dtype)
    k = idx.n_pages
    for src in ([7], [9, 7, 15, 2, 8], [1, 1, 14]):
        for masked in (False, True):
            masks, index = random_masks(idx, len(src), 3 + len(src)) if masked else (None, None)
            ws, wi, wc = reference(idx, src, k, masks, index)
            ts, ti, tc = host(idx.search_pages(src, k, masks, index))
            what = (dtype, src, masked)
            assert np.array_equal(tc, wc), what
            assert np.array_equal(ti, wi), what
            assert np.array_equal(bits(ts), bits(ws)), what
    # the float rows the first stages take are the same dequantised rows
    rows, lens = idx.page_rows([9, 0, 4])
    want = np.concatenate([dequantised(idx, p) for p in (9, 0, 4)])
    assert lens == [LENS[9], 0, LENS[4]]
    assert np.array_equal(rows[:sum(lens)].cpu().numpy(), want)


@pytest.mark.parametrize("dtype", ["bf16", "int8", "fp8", "binary"])
def test_zero_row_source_gets_nothing(dtype):
    idx = _index(dtype)
    ts, ti, tc = host(idx.search_pages([0, 7, 0], 5))
    assert list(tc) == [0, 5, 0]
    assert np.all(ti[[0, 2]] == -1) and np.all(np.isneginf(ts[[0, 2]]))
    assert ti[1, 0] in (7, len(PAGES) - 1)  # the page itself or its exact copy


def _i8_corpus():
    rng = np.random.default_rng(2)
    pages = [rng.integers(-127, 128, size=(n, 128)).astype(np.int8) for n in (5, 40, 0, 33, 300)]
    pages.append(np.full((1100, 128), 127, np.int8))   # a source past the bound
    pages.append(np.full((2, 128), 127, np.int8))
    pages.append(np.full((3, 128), -128, np.int8))
    pages.append(np.full((1, 128), 126, np.int8))
    return pages


def test_int8_is_exact_and_clamps():
    pages = _i8_corpus()
    lens = [len(p) for p in pages]
    packed = np.concatenate([np.concatenate([p, np.repeat(p[-1:], -len(p) % 32, axis=0)]) for p in pages if len(p)])
    idx = MaxSimIndex(dtype="int8")
    idx.append_packed(torch.from_numpy(packed.view(np.uint8)).to(DEV), lens)
    rows = np.concatenate(pages)
    off = orc.page_offsets(lens)
    src = [0, 1, 3, 4, 5, 7]
    k = idx.n_pages
    masks, index = random_masks(idx, len(src), 21)
    for masked in (False, True):
        ts, ti, tc = host(idx.search_pages(src, k, masks if masked else None, index if masked else None))
        mrows = masks.cpu().numpy().view(np.uint32)
        for i, p in enumerate(src):
            sums = orc.int8_maxsim_c(pages[p], rows, off).astype(np.int64)
            allow = None
            if masked and int(index[i]) >= 0:
                allow = np.unpackbits(mrows[int(index[i])].view(np.uint8), bitorder="little")[:idx.n_pages].astype(bool)
            ws, wi = orc.topk_np(i32_sum(sums), k, allow)
            n = len(wi)
            what = (p, masked)
            assert int(tc[i]) == n and np.array_equal(ti[i, :n], wi), what
            want = i32_reported(ws, idx.score_scale) / np.float32(lens[p])
            assert np.array_equal(bits(ts[i, :n]), bits(want)), what
    # the 1100-row +127 source passes 2^31 - 1 against both +127 pages: clamped, tied, lower id first
    ts, ti, tc = host(idx.search_pages([5], 3))
    assert list(ti[0, :2]) == [5, 6]
    assert bits(ts[0, 0]) == bits(ts[0, 1]) == bits(i32_reported(np.int64(2**31), idx.score_scale) / np.float32(1100))


def test_bf16_against_float64_page_maxsim():
    idx = _index("bf16")
    q = [orc.bf16_round_np(p) for p in PAGES]
    src = [LENS.index(n) for n in (0, 1, 31, 33, 1024, 1500)]
    k = 8
    ts, ti, tc = host(idx.search_pages(src, k))
    for i, p in enumerate(src):
        if LENS[p] == 0:
            assert tc[i] == 0
            continue
        want = np.array([page_sum(q[p], q[j], "bf16") / LENS[p] for j in range(len(PAGES))])
        got_ids = ti[i, :tc[i]]
        assert tc[i] == k
        err = np.abs(ts[i, :k] - want[got_ids]).max() / np.abs(want).max()
        assert err <= TOL["bf16"], (p, err)
        # nothing left out beats the k-th pick beyond the tolerance
        rest = np.setdiff1d(np.arange(len(PAGES)), got_ids)
        assert want[rest].max() <= ts[i, k - 1] + TOL["bf16"] * np.abs(want).max(), p


@pytest.mark.parametrize("dtype", ["bf16", "int8", "fp8", "binary"])
def test_host_tier_rerank_matches_hbm_and_gathers_only_candidates(dtype):
    hbm, hst = _index(dtype), _index(dtype, "host")
    src = [9, 8, 0, 3]
    rng = np.random.default_rng(4)
    cand = rng.integers(0, len(PAGES), size=(len(src), 9))
    cand[:, 2] = -1
    cand_dev = torch.from_numpy(cand).to(DEV)
    masks, index = random_masks(hbm, len(src), 8)
    for m, ix in ((None, None), (masks, index)):
        a = host(hbm.rerank_pages_batch(src, cand_dev, 6, m, ix))
        b = host(hst.rerank_pages_batch(src, cand_dev, 6, m, ix))
        for x, y in zip(a, b):
            assert np.array_equal(x.view(np.uint8), y.view(np.uint8)), (dtype, m is not None)
        st = hst.gather_stats()
        u = np.unique(cand[cand >= 0])
        pad = (hst.page_lens[u].astype(np.int64) + 31) // 32 * 32
        assert (st["unique_pages"], st["bytes"]) == (len(u), int(pad.sum()) * hst.row_bytes)
    # the rerank with every page as a candidate is the full scan
    every = torch.arange(len(PAGES), device=DEV).repeat(len(src), 1).contiguous()
    full = host(hbm.search_pages(src, 6))
    got = host(hst.rerank_pages_batch(src, every, 6))
    for x, y in zip(full, got):
        assert np.array_equal(x.view(np.uint8), y.view(np.uint8)), dtype
    with pytest.raises(nat.NativeError, match="host-resident"):
        hst.search_pages(src, 6)


@pytest.mark.parametrize("stage", ["fde", "sign"])
@pytest.mark.parametrize("tier", ["hbm", "host"])
@pytest.mark.parametrize("dtype", ["bf16", "int8"])
def test_two_stage_with_every_page_equals_exhaustive(stage, tier, dtype):
    from morphik_core_b200.fde import TwoStageIndex
    from morphik_core_b200.signs import SignTwoStageIndex

    two = (TwoStageIndex if stage == "fde" else SignTwoStageIndex)(dtype=dtype, tier=tier)
    two.add_pages(PAGES)
    src = [9, 0, 7, 4]
    ts, ti, tc = two.search_pages(src, 6, n_candidates=len(PAGES))
    want = host(_index(dtype).search_pages(src, 6))
    assert np.array_equal(tc, want[2]) and np.array_equal(ti, want[1]), (stage, tier, dtype)
    assert np.array_equal(bits(ts), bits(want[0]))
    names = {"fde": "encode_query_ms", "sign": "sign_candidates_ms"}[stage]
    assert names in two.last_timing_ms and "maxsim_rerank_ms" in two.last_timing_ms
    # per-source masks filter the rerank: the source itself is never returned
    words = []
    for p in src:
        allow = np.ones(len(PAGES), bool)
        allow[p] = False
        words.append(two.index.mask_from_pages(allow))
    ts, ti, tc = two.search_pages(src, 6, n_candidates=len(PAGES), allow_masks=np.stack(words))
    for i, p in enumerate(src):
        assert p not in ti[i, :tc[i]]


def test_refusals_launch_nothing():
    idx = _index("bf16")
    out = [torch.empty((2, 4), dtype=torch.float32, device=DEV), torch.empty((2, 4), dtype=torch.int64, device=DEV),
           torch.empty((2,), dtype=torch.int32, device=DEV)]
    ptrs = [ctypes.c_void_p(t.data_ptr()) for t in out]
    s = ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)
    cand = torch.zeros((2, 3), dtype=torch.int64, device=DEV)
    before = idx.launch_count()
    for ids, n in (([0, idx.n_pages], 2), ([-1, 0], 2), ([0, 1], 0), ([0, 1], -1)):
        a = nat.i64_array(ids)
        assert nat.lib.b200ms_search_pages_device(idx.h.ptr, a, n, 4, None, 0, None, ctypes.c_float(1), 0, *ptrs, s) == -1
        assert nat.lib.b200ms_rerank_pages_batch_device(idx.h.ptr, a, n, ctypes.c_void_p(cand.data_ptr()), 3, 4, None, 0,
                                                        None, ctypes.c_float(1), *ptrs, s) == -1
        assert nat.lib.b200ms_page_rows_device(idx.h.ptr, a, n, ctypes.c_float(1), ptrs[0], s) == -1
    a = nat.i64_array([0, 1])
    assert nat.lib.b200ms_search_pages_device(idx.h.ptr, a, 2, 0, None, 0, None, ctypes.c_float(1), 0, *ptrs, s) == -1
    assert nat.lib.b200ms_search_pages_device(idx.h.ptr, a, 2, 4, None, 1, None, ctypes.c_float(1), 0, *ptrs, s) == -1
    hst = _index("bf16", "host")
    h0 = hst.launch_count()
    assert nat.lib.b200ms_search_pages_device(hst.h.ptr, a, 2, 4, None, 0, None, ctypes.c_float(1), 0, *ptrs, s) == -3
    assert idx.launch_count() == before and hst.launch_count() == h0


@pytest.mark.parametrize("first", ["search_device", "search_pages"])
def test_in_flight_on_another_stream(first):
    """One handle: call A on stream 1 over a corpus large enough to still run, call B at once on stream 2; both results
    equal the same calls made alone."""
    rng = np.random.default_rng(31)
    pages = [_unit(rng, 512) for _ in range(1500)]
    idx = MaxSimIndex(dtype="bf16")
    idx.add_pages(pages)
    q = torch.from_numpy(np.concatenate([_unit(rng, 96) for _ in range(16)])).to(DEV)
    src = [3, 100, 1499]

    def call(which):
        return idx.search_device(q, [96] * 16, 10) if which == "search_device" else idx.search_pages(src, 10)

    second = "search_pages" if first == "search_device" else "search_device"
    alone = {w: host(call(w)) for w in (first, second)}
    torch.cuda.synchronize()
    s1, s2 = torch.cuda.Stream(), torch.cuda.Stream()
    with torch.cuda.stream(s1):
        a = call(first)
    with torch.cuda.stream(s2):
        b = call(second)
    torch.cuda.synchronize()
    for got, w in ((a, first), (b, second)):
        for x, y in zip(host(got), alone[w]):
            assert np.array_equal(x.view(np.uint8), y.view(np.uint8)), w


def test_store_chunks_like_a_stored_chunk():
    store = B200MultiVectorStore(mode="bf16", coalesce_queries=False)
    rng = np.random.default_rng(12)
    base = _unit(rng, 60)
    chunks = []
    for d in range(4):
        for c in range(3):
            e = base + np.float32(0.05 * (d + 1)) * _unit(rng, 60) if (d, c) != (0, 0) else base
            e = e / np.linalg.norm(e, axis=1, keepdims=True)  # unit rows, as the embedding model emits them
            chunks.append(DocumentChunk(document_id=f"d{d}", chunk_number=c, content="", embedding=e, metadata={}))
    asyncio.run(store.store_embeddings(chunks))
    res = asyncio.run(store.query_similar_to_chunks([("d0", 0), ("nope", 1), ("d0", 0), ("d2", 1)], k=20))
    assert len(res) == 2
    assert all(r.document_id != "d0" for r in res[0]) and len(res[0]) == 9
    assert [r.document_id for r in res[0][:3]] == ["d1"] * 3  # the nearest copies of the source
    assert all(r.document_id != "d2" for r in res[1])
    res = asyncio.run(store.query_similar_to_chunks([("d0", 0)], k=20, include_same_document=True))
    assert sorted((r.document_id, r.chunk_number) for r in res[0] if r.document_id == "d0") == [("d0", 1), ("d0", 2)]


def test_fde_first_stage_keeps_each_source_to_its_mask_row():
    """b200ms_topk_masked over the FDE scores: each source's candidates are exactly a b200ms_topk of its own mask row."""
    from morphik_core_b200.fde import TwoStageIndex

    two = TwoStageIndex(dtype="bf16")
    two.add_pages(PAGES)
    src = [9, 0, 7, 4, 12]
    rows, lens = two.index.page_rows(src)
    q = two._encode(None, (rows, nat.F32, lens))
    masks, index = random_masks(two.index, len(src), 17)
    got = host(two._scan(q, lens, 6, masks, index))
    for i in range(len(src)):
        row = int(index[i])
        want = host(two._scan(q[i:i + 1].contiguous(), lens[i:i + 1], 6, masks[row] if row >= 0 else None))
        for g, w in zip(got, want):
            assert np.array_equal(g[i:i + 1].view(np.uint8), w.view(np.uint8)), (i, row)


def _store_corpus(rng):
    """A 12-chunk document of near-copies of its chunk 0 (the source) and 5 other documents of 3 unit-row chunks each."""
    base = _unit(rng, 64)
    out = []
    for c in range(12):
        e = base if c == 0 else base + np.float32(0.05) * _unit(rng, 64)
        out.append(DocumentChunk(document_id="big", chunk_number=c, content="",
                                 embedding=e / np.linalg.norm(e, axis=1, keepdims=True), metadata={}))
    for d in range(5):
        for c in range(3):
            out.append(DocumentChunk(document_id=f"o{d}", chunk_number=c, content="", embedding=_unit(rng, 50), metadata={}))
    return out


@pytest.mark.parametrize("stage", ["fde", "sign"])
@pytest.mark.parametrize("tier", ["hbm", "host"])
def test_two_stage_store_with_fewer_candidates_than_the_source_document(stage, tier):
    """4 candidate slots, a source whose own document holds its 11 nearest chunks: the first stage must not spend its slots
    on pages the source may not return, so k = 5 chunks of other documents still come back, as in the exhaustive store."""
    kw = {"fde_candidates": 4} if stage == "fde" else {"sign_candidates": 4}
    store = B200MultiVectorStore(mode="bf16", coalesce_queries=False, corpus_tier=tier, **kw)
    exhaustive = B200MultiVectorStore(mode="bf16", coalesce_queries=False)
    for s_ in (store, exhaustive):
        asyncio.run(s_.store_embeddings(_store_corpus(np.random.default_rng(40))))
    res = asyncio.run(store.query_similar_to_chunks([("big", 0), ("o1", 2)], k=5))
    want = asyncio.run(exhaustive.query_similar_to_chunks([("big", 0), ("o1", 2)], k=5))
    assert [len(r) for r in res] == [len(r) for r in want] == [5, 5]
    assert all(c.document_id != "big" for c in res[0]) and all(c.document_id != "o1" for c in res[1])
    assert "maxsim_rerank_ms" in store.last_query_timing
    res = asyncio.run(store.query_similar_to_chunks([("big", 0)], k=5, include_same_document=True))
    assert [c.document_id for c in res[0]] == ["big"] * 5 and all(c.chunk_number != 0 for c in res[0])


def test_fde_page_search_in_flight_on_another_stream():
    """One handle: a two-stage page search (FDE scan, b200ms_topk_masked, rerank) on stream 1 and a full search at once on
    stream 2, then the reverse; every result equals the same call made alone."""
    from morphik_core_b200.fde import TwoStageIndex

    rng = np.random.default_rng(8)
    two = TwoStageIndex(dtype="bf16")
    two.add_pages([_unit(rng, 512) for _ in range(1500)])
    idx = two.index
    q = torch.from_numpy(np.concatenate([_unit(rng, 96) for _ in range(16)])).to(DEV)
    src = [3, 100, 1499]
    masks, index = random_masks(idx, len(src), 9)
    calls = {"pages": lambda: two.search_pages_device(src, 10, 50, masks, index)[:3],
             "search": lambda: idx.search_device(q, [96] * 16, 10)}
    alone = {w: host(f()) for w, f in calls.items()}
    for first, second in (("pages", "search"), ("search", "pages")):
        torch.cuda.synchronize()
        s1, s2 = torch.cuda.Stream(), torch.cuda.Stream()
        with torch.cuda.stream(s1):
            a = calls[first]()
        with torch.cuda.stream(s2):
            b = calls[second]()
        torch.cuda.synchronize()
        for got, w in ((a, first), (b, second)):
            for x, y in zip(host(got), alone[w]):
                assert np.array_equal(x.view(np.uint8), y.view(np.uint8)), (first, w)
