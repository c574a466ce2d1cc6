"""Relevance feedback on an H100 (run with -m gpu): b200ms_search_examples_device, b200ms_rerank_examples_batch_device and
b200ms_union_candidates_device through MaxSimIndex, the two first stages and the store.

- identity: one page example of weight 1 is search_pages bit for bit; one query example is search_device over T;
- fusion: mixed query and page examples, random positive and negative weights, several requests per call, sparse and dense
  masks, full scan and candidate lists, against the per-example rows of search_pages / search_device (k = every page)
  fused in numpy float32 in the stated order -- bit-identical ids, scores and counts on bf16, int8, fp8 and 1-bit;
- an independent oracle (tests/mmr_oracle.py's page sums): exact for int8 and 1-bit, float64 tolerance for bf16 and fp8;
- an int8 page example past the I32 bound fuses its clamped value;
- two-stage with every page a candidate equals the exhaustive call (FDE and signs, HBM and host tier); the union keeps
  first-occurrence order without repeats, and a page near only a negative example never becomes a candidate;
- the host tier gathers only the union's pages; refusals launch nothing; a call in flight on another stream; the store.
"""
import asyncio
import ctypes

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

torch = pytest.importorskip("torch")
if not torch.cuda.is_available():  # pragma: no cover - the gpu marker normally deselects these on CPU boxes
    pytest.skip("CUDA device required", allow_module_level=True)

from mmr_oracle import page_sum, quantise_rows  # noqa: E402
from morphik_core_b200 import _native as nat  # noqa: E402
from morphik_core_b200.index import MaxSimIndex  # noqa: E402
from morphik_core_b200.models import DocumentChunk  # noqa: E402
from morphik_core_b200.store import B200MultiVectorStore  # noqa: E402
from oracle.scoring import TOL, i32_reported  # noqa: E402

DEV = torch.device("cuda", 0)
LENS = [0, 1, 31, 32, 33, 64, 65, 200, 1024, 300, 17, 90, 3, 128, 40]
DTYPES = ["bf16", "int8", "fp8", "binary"]
KIND = {"bf16": "bf16", "int8": "int8", "fp8": "fp8", "binary": "bits"}


def _unit(rng, n):
    x = rng.standard_normal((n, 128)).astype(np.float32)
    return x / np.maximum(np.linalg.norm(x, axis=1, keepdims=True), 1e-9)


def _pages(seed=5, lens=LENS):
    rng = np.random.default_rng(seed)
    pages = [_unit(rng, n) for n in lens]
    pages.append(pages[7].copy())  # an exact copy: ties broken by page id
    return pages


PAGES = _pages()
_IDX = {}


def _index(dtype, tier="hbm", corpus="mixed"):
    key = (dtype, tier, corpus)
    if key not in _IDX:
        idx = MaxSimIndex(dtype=dtype, tier=tier)
        if corpus == "mixed":
            idx.add_pages(PAGES)
        else:  # 3000 short pages: a fusion grid of many CTAs, sliced selections
            rng = np.random.default_rng(77)
            idx.add_pages([_unit(rng, int(n)) for n in rng.integers(1, 12, size=3000)])
        idx._attach()
        _IDX[key] = idx
    return _IDX[key]


def bits(x):
    return np.ascontiguousarray(x, np.float32).view(np.uint32)


def host(ts):
    return tuple(t.cpu().numpy() for t in ts)


def _queries(seed, lens):
    rng = np.random.default_rng(seed)
    return [_unit(rng, n) for n in lens]


def _qdev(queries):
    return torch.from_numpy(np.concatenate(queries) if queries else np.zeros((0, 128), np.float32)).to(DEV)


def example_rows(idx, queries, pages):
    """Each example's score of every page: page examples from search_pages, query examples from search_device / T
    (float32), with k = every page; None for an example without rows."""
    n = idx.n_pages
    rows = []
    for q in queries:
        if len(q) == 0:
            rows.append(None)
            continue
        ts, ti, tc = host(idx.search_device(_qdev([q]), [len(q)], n))
        r = np.zeros(n, np.float32)
        r[ti[0, :tc[0]]] = ts[0, :tc[0]] / np.float32(len(q))
        rows.append(r)
    for p in pages:
        if idx.page_lens[p] == 0:
            rows.append(None)
            continue
        ts, ti, tc = host(idx.search_pages([p], n))
        assert tc[0] == n
        r = np.zeros(n, np.float32)
        r[ti[0]] = ts[0]
        rows.append(r)
    return rows


def fuse(rows, ex_req, weights, n_req):
    """The header's fused rows in numpy float32: acc = 0; acc = acc + w * s in example order (no FMA), then + 0 (the
    selection's key: -0 ranks and reports as +0)."""
    n = next(len(r) for r in rows if r is not None)
    out = np.zeros((n_req, n), np.float32)
    for r, e_req, w in zip(rows, ex_req, np.asarray(weights, np.float32)):
        if r is not None:
            out[e_req] = out[e_req] + w * r
    return out + np.float32(0)


def select(scores, allow, k, ids=None):
    """b200ms_topk's order over one fused row: allowed items by (score DESC, position ASC); ids maps positions to pages."""
    pos = np.flatnonzero(allow)
    order = pos[np.lexsort((pos, -scores[pos].astype(np.float64)))][:k]
    return scores[order], (order if ids is None else ids[order]), len(order)


def allow_rows(idx, masks, index, n_req):
    n = idx.n_pages
    if masks is None:
        return [np.ones(n, bool)] * n_req
    m = masks.cpu().numpy().view(np.uint32)
    out = []
    for r in range(n_req):
        row = int(index[r])
        out.append(np.ones(n, bool) if row < 0 else
                   np.unpackbits(m[row].view(np.uint8), bitorder="little")[:n].astype(bool))
    return out


def check(got, fused, allows, k, cands=None):
    ts, ti, tc = got
    for r in range(len(allows)):
        if cands is None:
            ws, wi, wc = select(fused[r], allows[r], k)
        else:  # slot-wise: valid slots of r's list whose page r may return
            c = cands[r]
            ok = np.array([0 <= p < len(allows[r]) and allows[r][p] for p in c])
            ws, wi, wc = select(fused[r][np.where(c >= 0, c, 0)], ok, k, c)
        assert tc[r] == wc, r
        assert np.array_equal(ti[r, :wc], wi), (r, ti[r, :wc], wi)
        assert np.array_equal(bits(ts[r, :wc]), bits(ws)), r
        assert np.all(ti[r, wc:] == -1)


def random_request_masks(idx, n_req, seed, dense):
    rng = np.random.default_rng(seed)
    fracs = (0.9, 0.6) if dense else (0.08, 0.02)
    words = [idx.mask_from_pages(rng.random(idx.n_pages) < f) for f in fracs]
    masks = torch.from_numpy(np.stack(words).view(np.int32)).to(DEV)
    index = torch.tensor([r % 3 - 1 for r in range(n_req)], dtype=torch.int32, device=DEV)
    return masks, index


def _batch(idx, seed):
    """Three requests mixing query and page examples, with a zero-row page and a zero-token query in the mix."""
    rng = np.random.default_rng(seed)
    queries = _queries(seed, [20, 0, 33, 70])
    n = idx.n_pages
    pages = [int(p) for p in rng.integers(0, n, size=5)] + ([0] if n == len(PAGES) else [1])
    ex_req = [0, 1, 2, 1, 2, 0, 1, 1, 2, 0]
    weights = [1.0, 0.75, 2.0, -0.3, 1.0, -1.5, 0.4, -0.6, -0.25, 0.5]
    weights = [np.float32(w * (1 + 0.1 * rng.standard_normal())) for w in weights]
    return queries, pages, ex_req, weights, 3


@pytest.mark.parametrize("dtype", DTYPES)
def test_identity_with_search_pages_and_search_device(dtype):
    idx = _index(dtype)
    n = idx.n_pages
    for p in (7, 9, 4):
        want = host(idx.search_pages([p], 6))
        got = host(idx.search_examples(None, [], [p], [0], [1.0], 1, 6))
        for x, y in zip(got, want):
            assert np.array_equal(x.view(np.uint8), y.view(np.uint8)), (dtype, p)
    q = _queries(3, [29])
    ts, ti, tc = host(idx.search_device(_qdev(q), [29], n))
    scores = ts[0] / np.float32(29)
    ws, wi, wc = select(np.array([scores[list(ti[0]).index(p)] for p in range(n)], np.float32) + np.float32(0),
                        np.ones(n, bool), n)
    got = host(idx.search_examples(_qdev(q), [29], [], [0], [1.0], 1, n))
    assert got[2][0] == wc and np.array_equal(got[1][0], wi) and np.array_equal(bits(got[0][0]), bits(ws)), dtype


@pytest.mark.parametrize("corpus", ["mixed", "many"])
@pytest.mark.parametrize("dtype", DTYPES)
def test_fusion_is_exact(dtype, corpus):
    if corpus == "many" and dtype in ("fp8", "binary"):
        pytest.skip("the many-page corpus runs on bf16 and int8")
    idx = _index(dtype, corpus=corpus)
    n = idx.n_pages
    queries, pages, ex_req, weights, n_req = _batch(idx, 11)
    rows = example_rows(idx, queries, pages)
    fused = fuse(rows, ex_req, weights, n_req)
    q = _qdev(queries)
    lens = [len(x) for x in queries]
    k = min(n, 40)
    for dense in (None, True, False):
        masks, index = (None, None) if dense is None else random_request_masks(idx, n_req, 5, dense)
        allows = allow_rows(idx, masks, index, n_req)
        got = host(idx.search_examples(q, lens, pages, ex_req, weights, n_req, k, masks, index, id_base=0))
        check(got, fused, allows, k)
        # candidate mode: one list per request with unused slots and a repeated page
        rng = np.random.default_rng(6)
        cands = rng.integers(0, n, size=(n_req, 37))
        cands[:, 3] = -1
        cands[:, 5] = cands[:, 4]
        got = host(idx.rerank_examples_batch(q, lens, pages, ex_req, weights, n_req, torch.from_numpy(cands).to(DEV), 12,
                                             masks, index))
        check(got, fused, allows, 12, cands)
    # id_base shifts the reported ids only
    a = host(idx.search_examples(q, lens, pages, ex_req, weights, n_req, 5))
    b = host(idx.search_examples(q, lens, pages, ex_req, weights, n_req, 5, id_base=1000))
    assert np.array_equal(np.where(a[1] >= 0, a[1] + 1000, -1), b[1]) and np.array_equal(bits(a[0]), bits(b[0]))


@pytest.mark.parametrize("dtype", DTYPES)
def test_against_independent_page_sums(dtype):
    idx = _index(dtype)
    kind = KIND[dtype]
    n = idx.n_pages
    qp = [quantise_rows(p, kind) for p in PAGES]
    ex_pages, weights = [9, 4, 13], [0.5, 1.0, -0.75]
    ts, ti, tc = host(idx.search_examples(None, [], ex_pages, [0, 0, 0], weights, 1, n))
    assert tc[0] == n
    exact = kind in ("int8", "bits")
    want = np.zeros(n, np.float32 if exact else np.float64)
    for p, w in zip(ex_pages, weights):
        sums = [page_sum(qp[p], qp[j], kind) for j in range(n)]
        if exact:
            s = np.array([i32_reported(np.int64(x), idx.score_scale) for x in sums], np.float32) / np.float32(LENS[p])
            want = want + np.float32(w) * s
        else:
            want += w * np.array(sums) * idx.score_scale / LENS[p]
    got = np.empty(n, np.float32)
    got[ti[0]] = ts[0]
    if exact:
        assert np.array_equal(bits(got), bits(want + np.float32(0))), dtype
    else:
        assert np.abs(got - want).max() <= TOL[kind] * np.abs(want).max() * 4, dtype


def test_int8_example_past_the_bound_fuses_its_clamped_value():
    pages = [np.full((1100, 128), 127, np.int8), np.full((2, 128), 127, np.int8), np.full((3, 128), -128, np.int8),
             np.full((5, 128), 1, np.int8)]
    lens = [len(p) for p in pages]
    packed = np.concatenate([np.concatenate([p, np.repeat(p[-1:], -len(p) % 32, axis=0)]) for p in pages])
    idx = MaxSimIndex(dtype="int8")
    idx.append_packed(torch.from_numpy(packed.view(np.uint8)).to(DEV), lens)
    ts, ti, tc = host(idx.search_examples(None, [], [0, 3], [0, 0], [1.0, -0.5], 1, 4))
    clamp = i32_reported(np.int64(2**31), idx.score_scale) / np.float32(1100)  # 1100 * 128 * 127^2 > 2^31 - 1
    got = dict(zip(ti[0].tolist(), ts[0]))
    # page 1 (+127 rows): the clamped first term, then the small page example's term
    s3 = i32_reported(np.int64(5 * 128 * 127), idx.score_scale) / np.float32(5)
    want1 = np.float32(0) + np.float32(1.0) * clamp + np.float32(-0.5) * s3
    assert bits(got[1]) == bits(want1)
    assert list(ti[0, :2]) == [0, 1]  # pages 0 and 1 tie on the clamped term and on the second: lower id first
    assert bits(got[0]) == bits(got[1])


def test_union_keeps_first_occurrence_without_repeats():
    idx = _index("bf16")
    cand = torch.tensor([[5, 3, -1, 5, 9], [3, 7, 2, 11, -1], [1, 1, 1, 1, 1], [-1, -1, -1, -1, -1], [14, 0, 2, 0, 6]],
                        dtype=torch.int64, device=DEV)
    out = idx.union_candidates(cand, [0, 2, 2, 4, 5]).cpu().numpy()
    assert out.shape == (4, 10)
    assert out[0].tolist() == [5, 3, 9, 7, 2, 11] + [-1] * 4
    assert out[1].tolist() == [-1] * 10
    assert out[2].tolist() == [1] + [-1] * 9
    assert out[3].tolist() == [14, 0, 2, 6] + [-1] * 6
    assert idx.union_candidates(cand, [0, 2, 2, 4, 5], width=2).cpu().numpy()[0].tolist() == [5, 3]
    # many long lists: every id once, in first-occurrence order
    rng = np.random.default_rng(3)
    big = rng.integers(-3, 5000, size=(7, 4096))
    out = idx.union_candidates(torch.from_numpy(big).to(DEV), [0, 3, 7]).cpu().numpy()
    for r, (a, b) in enumerate(((0, 3), (3, 7))):
        flat = big[a:b].reshape(-1)
        _, first = np.unique(flat[flat >= 0], return_index=True)
        want = flat[flat >= 0][np.sort(first)]
        assert np.array_equal(out[r, :len(want)], want) and np.all(out[r, len(want):] == -1), r


def _two(stage, dtype, tier):
    from morphik_core_b200.fde import TwoStageIndex
    from morphik_core_b200.signs import SignTwoStageIndex

    two = (TwoStageIndex if stage == "fde" else SignTwoStageIndex)(dtype=dtype, tier=tier)
    two.add_pages(PAGES)
    return two


@pytest.mark.parametrize("stage", ["fde", "sign"])
@pytest.mark.parametrize("tier", ["hbm", "host"])
@pytest.mark.parametrize("dtype", ["bf16", "int8"])
def test_two_stage_with_every_page_equals_exhaustive(stage, tier, dtype):
    two = _two(stage, dtype, tier)
    queries = _queries(21, [25, 40])
    pages, ex_req = [9, 4, 13, 2], [0, 1, 0, 1, 1, 0]
    weights = [1.0, 0.5, 0.5, -1.0, 0.8, -0.2]
    rng = np.random.default_rng(8)
    words = np.stack([two.index.mask_from_pages(rng.random(len(PAGES)) < 0.7) for _ in range(2)])
    for w in (None, words):
        ts, ti, tc = two.search_examples(queries, pages, ex_req, weights, 2, 6, n_candidates=len(PAGES), allow_masks=w)
        mdev = None if w is None else torch.from_numpy(np.ascontiguousarray(w).view(np.int32)).to(DEV)
        idev = None if w is None else torch.arange(2, dtype=torch.int32, device=DEV)
        want = host(_index(dtype).search_examples(_qdev(queries), [25, 40], pages, ex_req, weights, 2, 6, mdev, idev))
        assert np.array_equal(tc, want[2]) and np.array_equal(ti, want[1]), (stage, tier, dtype, w is None)
        assert np.array_equal(bits(ts), bits(want[0]))
        if tier == "host" and w is None:  # every page is a candidate of both lists, and each crossed PCIe once
            st = two.index.gather_stats()
            assert int((two.index.page_lens > 0).sum()) <= st["unique_pages"] <= len(PAGES)
    names = {"fde": "encode_query_ms", "sign": "sign_candidates_ms"}[stage]
    assert names in two.last_timing_ms and "maxsim_rerank_ms" in two.last_timing_ms


@pytest.mark.parametrize("stage", ["fde", "sign"])
def test_a_page_near_only_a_negative_never_becomes_a_candidate(stage):
    from morphik_core_b200.fde import TwoStageIndex
    from morphik_core_b200.signs import SignTwoStageIndex

    rng = np.random.default_rng(50)
    a, b = _unit(rng, 40), _unit(rng, 40)
    far = [_unit(rng, 40) for _ in range(30)]
    near_a = [(a + np.float32(0.05) * _unit(rng, 40)) for _ in range(3)]
    near_b = [(b + np.float32(0.05) * _unit(rng, 40)) for _ in range(3)]
    pages = [a, b] + near_a + near_b + far  # 0 = a, 1 = b, 2..4 near a, 5..7 near b
    two = (TwoStageIndex if stage == "fde" else SignTwoStageIndex)(dtype="bf16", tier="host")
    two.add_pages([p / np.linalg.norm(p, axis=1, keepdims=True) for p in pages])
    ts, ti, tc, _ = two.search_examples_device([], [0, 1], [0, 0], [1.0, -1.0], 1, 3, n_candidates=4)
    torch.cuda.synchronize()
    st = two.index.gather_stats()
    ids = set(ti.cpu().numpy()[0, :int(tc[0])].tolist())
    assert st["unique_pages"] <= 4 and not ids & {1, 5, 6, 7}
    assert len(ids) == 3 and ids <= {0, 2, 3, 4}


@pytest.mark.parametrize("dtype", DTYPES)
def test_host_tier_rerank_matches_hbm_and_gathers_only_the_union(dtype):
    hbm, hst = _index(dtype), _index(dtype, "host")
    queries, pages, ex_req, weights, n_req = _batch(hbm, 13)
    q, lens = _qdev(queries), [len(x) for x in queries]
    rng = np.random.default_rng(4)
    lists = torch.from_numpy(rng.integers(-1, len(PAGES), size=(5, 6))).to(DEV)
    union = hbm.union_candidates(lists, [0, 2, 3, 5])
    masks, index = random_request_masks(hbm, n_req, 9, True)
    for m, ix in ((None, None), (masks, index)):
        a = host(hbm.rerank_examples_batch(q, lens, pages, ex_req, weights, n_req, union, 7, m, ix))
        b = host(hst.rerank_examples_batch(q, lens, pages, ex_req, weights, n_req, union, 7, m, ix))
        for x, y in zip(a, b):
            assert np.array_equal(x.view(np.uint8), y.view(np.uint8)), (dtype, m is not None)
        st = hst.gather_stats()
        u = np.unique(union.cpu().numpy())
        u = u[u >= 0]
        pad = (hst.page_lens[u].astype(np.int64) + 31) // 32 * 32
        assert (st["unique_pages"], st["bytes"]) == (len(u), int(pad.sum()) * hst.row_bytes)
    with pytest.raises(nat.NativeError, match="host-resident"):
        hst.search_examples(q, lens, pages, ex_req, weights, n_req, 4)


def test_refusals_launch_nothing():
    idx = _index("bf16")
    hst = _index("bf16", "host")
    out = [torch.empty((2, 4), dtype=torch.float32, device=DEV), torch.empty((2, 4), dtype=torch.int64, device=DEV),
           torch.empty((2,), dtype=torch.int32, device=DEV)]
    ptrs = [ctypes.c_void_p(t.data_ptr()) for t in out]
    s = ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)
    cand = torch.zeros((2, 3), dtype=torch.int64, device=DEV)
    q = _qdev(_queries(1, [8]))
    qp = ctypes.c_void_p(q.data_ptr())
    f = ctypes.c_float(1)
    n = idx.n_pages
    #          n_qe, pages, ex_req, weights, n_req, k, n_masks
    bad = [(0, [], [], [], 1, 4, 0),                       # no example
           (0, [1], [0], [-1.0], 1, 4, 0),                 # no positive example
           (0, [1, 2], [0, 1], [1.0, -1.0], 2, 4, 0),      # request 1 has no positive
           (0, [1], [0], [0.0], 1, 4, 0),                  # zero weight
           (0, [1], [0], [float("nan")], 1, 4, 0),         # non-finite weight
           (0, [1], [0], [float("inf")], 1, 4, 0),
           (0, [1], [1], [1.0], 1, 4, 0),                  # ex_req out of range
           (0, [1], [-1], [1.0], 1, 4, 0),
           (0, [n], [0], [1.0], 1, 4, 0),                  # page out of range
           (0, [-1], [0], [1.0], 1, 4, 0),
           (0, [1], [0], [1.0], 1, 0, 0),                  # bad k
           (0, [1], [0], [1.0], 1, 4097, 0),
           (0, [1], [0], [1.0], 1, 4, 1),                  # masks without their matrix
           (1, [1], [0, 0], [1.0, 1.0], 0, 4, 0)]          # no request
    for h, before in ((idx, idx.launch_count()), (hst, hst.launch_count())):
        for n_qe, pages, req, w, n_req, k, n_masks in bad:
            args = (qp, nat.F32, nat.i32_array([8] * n_qe), n_qe, nat.i64_array(pages), len(pages), nat.i32_array(req),
                    nat.f32_array(w), n_req)
            if h is idx:
                assert nat.lib.b200ms_search_examples_device(h.h.ptr, *args, k, None, n_masks, None, f, f, 0, *ptrs, s) == -1
            assert nat.lib.b200ms_rerank_examples_batch_device(h.h.ptr, *args, ctypes.c_void_p(cand.data_ptr()), 3, k, None,
                                                               n_masks, None, f, f, *ptrs, s) == -1
        assert h.launch_count() == before
    ok = (qp, nat.F32, nat.i32_array([8]), 1, nat.i64_array([2]), 1, nat.i32_array([0, 0]), nat.f32_array([1.0, -1.0]), 1)
    h0 = hst.launch_count()
    assert nat.lib.b200ms_search_examples_device(hst.h.ptr, *ok, 4, None, 0, None, f, f, 0, *ptrs, s) == -3
    assert hst.launch_count() == h0
    before = idx.launch_count()
    o = ctypes.c_void_p(cand.data_ptr())
    c = ctypes.c_void_p(cand.data_ptr())
    for lists, n_cand, off, n_req, width in ((2, 3, [0, 1], 1, 4), (2, 3, [1, 2], 1, 4), (2, 3, [0, 2, 1], 2, 4),
                                            (2, 3, [0, 2], 0, 4), (2, 0, [0, 2], 1, 4), (2, 3, [0, 2], 1, 0)):
        assert nat.lib.b200ms_union_candidates_device(idx.h.ptr, c, lists, n_cand, nat.i32_array(off), n_req, o, width, s) == -1
    assert idx.launch_count() == before


@pytest.mark.parametrize("first", ["search_device", "search_examples", "rerank_examples"])
def test_in_flight_on_another_stream(first):
    """One handle: call A on stream 1 over a corpus large enough to still run, call B at once on stream 2; both results
    equal the same calls made alone."""
    rng = np.random.default_rng(31)
    idx = MaxSimIndex(dtype="bf16")
    idx.add_pages([_unit(rng, 512) for _ in range(1500)])
    q = torch.from_numpy(np.concatenate([_unit(rng, 96) for _ in range(16)])).to(DEV)
    qe = torch.from_numpy(_unit(rng, 30)).to(DEV)
    lists = torch.from_numpy(rng.integers(0, 1500, size=(2, 300))).to(DEV)
    calls = {"search_device": lambda: idx.search_device(q, [96] * 16, 10),
             "search_examples": lambda: idx.search_examples(qe, [30], [3, 100, 1499], [0, 0, 1, 1], [1.0, -0.5, 1.0, 0.3], 2,
                                                            10),
             "rerank_examples": lambda: idx.rerank_examples_batch(qe, [30], [3, 1499], [1, 0, 1], [1.0, 1.0, -0.5], 2,
                                                                  idx.union_candidates(lists, [0, 1, 2]), 10)}
    alone = {w: host(f()) for w, f in calls.items()}
    for second in calls:
        if second == first:
            continue
        torch.cuda.synchronize()
        s1, s2 = torch.cuda.Stream(), torch.cuda.Stream()
        with torch.cuda.stream(s1):
            a = calls[first]()
        with torch.cuda.stream(s2):
            b = calls[second]()
        torch.cuda.synchronize()
        for got, w in ((a, first), (b, second)):
            for x, y in zip(host(got), alone[w]):
                assert np.array_equal(x.view(np.uint8), y.view(np.uint8)), (first, second, w)


def _store_chunks(rng):
    """Document "a": near-copies of base_a; document "b": near-copies of base_b; documents o*: unrelated."""
    base_a, base_b = _unit(rng, 50), _unit(rng, 50)
    out = []
    for d, base in (("a", base_a), ("b", base_b)):
        for c in range(4):
            e = base + np.float32(0.1 * (c + 1)) * _unit(rng, 50)
            out.append(DocumentChunk(document_id=d, chunk_number=c, content="",
                                     embedding=e / np.linalg.norm(e, axis=1, keepdims=True), metadata={}))
    for d in range(4):
        out.append(DocumentChunk(document_id=f"o{d}", chunk_number=0, content="", embedding=_unit(rng, 40), metadata={}))
    return out, base_a


@pytest.mark.parametrize("mode", ["exhaustive", "fde", "sign"])
def test_store_feedback(mode):
    kw = {"fde": {"fde_candidates": 6}, "sign": {"sign_candidates": 6}}.get(mode, {})
    store = B200MultiVectorStore(mode="bf16", coalesce_queries=False, **kw)
    chunks, base_a = _store_chunks(np.random.default_rng(9))
    asyncio.run(store.store_embeddings(chunks))
    res = asyncio.run(store.query_similar_with_feedback(None, k=3, positive_chunks=[("a", 0)]))
    assert [c.document_id for c in res] == ["a"] * 3 and all(c.chunk_number != 0 for c in res)
    # liking a chunk of "a" and disliking one of "b": "b" ranks last
    res = asyncio.run(store.query_similar_with_feedback(base_a, k=20, positive_chunks=[("a", 1)],
                                                        negative_chunks=[("b", 0), ("nope", 1)]))
    ids = [(c.document_id, c.chunk_number) for c in res]
    assert ("a", 1) not in ids and ("b", 0) not in ids and [d for d, _ in ids[:3]] == ["a"] * 3
    if mode == "exhaustive":
        assert len(ids) == 10 and [d for d, _ in ids[-3:]] == ["b"] * 3
    else:
        assert "maxsim_rerank_ms" in store.last_query_timing
    assert asyncio.run(store.query_similar_with_feedback(None, k=3, negative_chunks=[("a", 0)])) == []
    with pytest.raises(ValueError):
        asyncio.run(store.query_similar_with_feedback(base_a, k=3, positive_chunks=[("a", 1)], negative_chunks=[("a", 1)]))
