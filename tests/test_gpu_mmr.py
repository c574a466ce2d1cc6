"""b200ms_mmr_device / MaxSimIndex.mmr / B200MultiVectorStore.query_similar_mmr on an H100 (run with -m gpu).

For bf16, int8, fp8 and binary corpora, on the HBM tier and the host tier: the page-to-page sims against the numpy oracle
(tests/mmr_oracle.py; oracle/scoring.py TOL for the float kinds, exact for int8 and binary) over page lengths 0 .. 1030 with
the 64-row tile edges and the corpus's last page; the pick order against greedy() replayed on the device's own rel and
sims, with no tolerance; lambda = 1 against the flat ranking bit for bit, also on pages holding +-inf; batches of lists with
unused and repeated slots; crafted non-finite pages; an int8 pair whose row sum passes int32; refusals that launch nothing;
determinism; host tier == HBM tier bit for bit; a planted store of near-copies; and a call in flight on another stream.
"""
import asyncio
import ctypes

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

torch = pytest.importorskip("torch")
if not torch.cuda.is_available():  # pragma: no cover - the gpu marker normally deselects these on CPU boxes
    pytest.skip("CUDA device required", allow_module_level=True)

from mmr_oracle import greedy, page_sims, quantise_rows, relevance, valid_slots  # noqa: E402
from morphik_core_b200 import _native as nat  # noqa: E402
from morphik_core_b200.index import MaxSimIndex  # noqa: E402
from morphik_core_b200.models import DocumentChunk  # noqa: E402
from morphik_core_b200.store import B200MultiVectorStore  # noqa: E402
from oracle.scoring import TOL  # noqa: E402

KIND = {"bf16": "bf16", "int8": "int8", "fp8": "fp8", "binary": "bits"}
DTYPES = list(KIND)
PLENS = [0, 1, 31, 32, 33, 63, 64, 65, 1024, 1030]
DEV = torch.device("cuda", 0)


def _unit(rng, n):
    x = rng.standard_normal((n, 128)).astype(np.float32)
    return x / np.maximum(np.linalg.norm(x, axis=1, keepdims=True), 1e-9)


def _corpus(seed=11):
    """PLENS pages, a near-copy of the 65-row page, an exact copy of the 33-row page, random pages, and a 65-row page last
    (its second 64-row tile runs 63 rows past the end of the corpus)."""
    rng = np.random.default_rng(seed)
    pages = [_unit(rng, n) for n in PLENS]
    near = pages[PLENS.index(65)] + np.float32(0.02) * _unit(rng, 65)
    pages.append(near / np.linalg.norm(near, axis=1, keepdims=True))
    pages.append(pages[PLENS.index(33)].copy())
    pages += [_unit(rng, int(n)) for n in rng.integers(1, 200, size=4)]
    pages.append(_unit(rng, 65))
    return pages


PAGES = _corpus()
N_PAGES = len(PAGES)
_INDEXES = {}


def _index(dtype, tier="hbm", pages=None, key=None):
    key = (key or "main", dtype, tier)
    if key not in _INDEXES:
        idx = MaxSimIndex(dtype=dtype, tier=tier)
        idx.add_pages(PAGES if pages is None else pages)
        idx._attach()
        _INDEXES[key] = idx
    return _INDEXES[key]


def _lists(n_q, seed, n_pages=N_PAGES, n=None):
    """Per-query lists: every page (or n random ones), -1, an id past the corpus, a repeated page."""
    rng = np.random.default_rng(seed)
    rows = []
    for _ in range(n_q):
        base = list(range(n_pages)) if n is None else [int(x) for x in rng.integers(0, n_pages, size=n - 3)]
        lst = base + [-1, n_pages + 5, base[len(base) // 2]]
        rng.shuffle(lst)
        rows.append(lst)
    return np.asarray(rows, dtype=np.int64)


def _scores(shape, seed):
    return np.random.default_rng(seed).standard_normal(shape).astype(np.float32)


def run_mmr(idx, ids, scores, q_lens, k, lam, with_sims=True):
    """MaxSimIndex.mmr on host arrays -> host arrays (ids, scores, counts, sims or None)."""
    ids_d = torch.from_numpy(np.ascontiguousarray(ids)).to(DEV)
    sc_d = torch.from_numpy(np.ascontiguousarray(scores)).to(DEV)
    out = idx.mmr(ids_d, sc_d, q_lens, k, lam, with_sims=with_sims)
    torch.cuda.synchronize()
    host = [t.cpu().numpy() for t in out]
    return host if with_sims else host + [None]


def first_slot(ids_row, pid):
    return int(np.flatnonzero(ids_row == pid)[0])


def check_picks(ids, scores, q_lens, k, lam, got, n_pages):
    """out_ids == greedy() replayed on the device's own rel and sims; scores bit for bit; counts; -1 / -inf past count."""
    gi, gs, gc, sims = got
    for q in range(ids.shape[0]):
        valid = valid_slots(ids[q], n_pages)
        n = ids.shape[1]
        m = np.full((n, n), np.nan, np.float32)
        for i in range(int(gc[q])):
            m[:, first_slot(ids[q], gi[q, i])] = sims[q, i]
        picks = greedy(relevance(scores[q], q_lens[q]), m, k, lam, valid)
        assert int(gc[q]) == len(picks) == min(k, int(valid.sum())), (q, int(gc[q]), len(picks))
        assert gi[q, :len(picks)].tolist() == ids[q, picks].tolist(), (q, gi[q, :len(picks)].tolist(), ids[q, picks].tolist())
        assert gs[q, :len(picks)].view(np.uint32).tolist() == scores[q, picks].view(np.uint32).tolist(), q
        assert (gi[q, len(picks):] == -1).all() and np.isneginf(gs[q, len(picks):]).all(), q


def check_sims(kind, ids, got, qpages, scale, slots=None):
    """sims against the oracle: the live slots of each pick row, -inf elsewhere.  slots: check only these (large lists)."""
    gi, _, gc, sims = got
    exact = kind in ("int8", "bits")
    tol = TOL["binary" if kind == "bits" else kind]
    for q in range(ids.shape[0]):
        valid = valid_slots(ids[q], len(qpages))
        want_all = {}
        live = valid.copy()
        for i in range(sims.shape[1]):
            if i < int(gc[q]):
                s = first_slot(ids[q], gi[q, i])
                live[s] = False
            else:
                live[:] = False
            cols = range(ids.shape[1]) if slots is None else slots
            for j in cols:
                g = sims[q, i, j]
                if not live[j]:
                    assert np.isneginf(g), (q, i, j, g)
                    continue
                pair = (int(ids[q, j]), int(ids[q, s]))
                if pair not in want_all:
                    want_all[pair] = page_sims([qpages[pair[0]], qpages[pair[1]]], np.array([0, 1]), kind, scale)[0, 1]
                w = want_all[pair]
                if exact:
                    assert g == np.float32(w), (q, i, j, g, w)
                elif np.isnan(w) or np.isinf(w):
                    assert (np.isnan(g) and np.isnan(w)) or g == w, (q, i, j, g, w)
                else:
                    assert abs(float(g) - w) <= tol * max(abs(w), 1.0), (q, i, j, float(g), w)


def _qpages(dtype, pages=None):
    return [quantise_rows(p, KIND[dtype]) for p in (PAGES if pages is None else pages)]


@pytest.mark.parametrize("tier", ["hbm", "host"])
@pytest.mark.parametrize("dtype", DTYPES)
def test_sims_and_picks_match_the_oracle(dtype, tier):
    idx = _index(dtype, tier)
    ids = _lists(3, seed=5)
    scores = _scores(ids.shape, seed=6)
    scores[2, 4] = np.nan  # a NaN score ranks first
    q_lens = [7, 0, 129]
    qp = _qpages(dtype)
    for lam in (0.5, 0.0, 0.3):
        got = run_mmr(idx, ids, scores, q_lens, ids.shape[1], lam)
        check_picks(ids, scores, q_lens, ids.shape[1], lam, got, N_PAGES)
        if lam == 0.5:
            check_sims(KIND[dtype], ids, got, qp, idx.score_scale)
        if tier == "host":  # bit-identical to the HBM tier
            ref = run_mmr(_index(dtype, "hbm"), ids, scores, q_lens, ids.shape[1], lam)
            for a, b in zip(got, ref):
                assert np.array_equal(a.view(np.uint8), b.view(np.uint8))
            assert idx.gather_stats()["rounds"] == 1


@pytest.mark.parametrize("dtype", ["bf16", "int8"])
@pytest.mark.parametrize("n", [1, 2, 33, 100, 1000])
def test_batches(dtype, n):
    rng = np.random.default_rng(n)
    pages = [_unit(rng, int(x)) for x in rng.integers(0, 70, size=1100)]
    pages[3] = pages[7].copy()
    idx = _index(dtype, pages=pages, key=f"batch{n}")
    n_q = 2 if n == 1000 else 3
    ids = _lists(n_q, seed=n, n_pages=len(pages), n=max(n, 4))[:, :n] if n >= 4 else \
        np.array([[int(rng.integers(0, len(pages))) for _ in range(n)] for _ in range(n_q)], np.int64)
    if n >= 2:
        ids[0, -1] = ids[0, 0]  # a repeated slot
        ids[1, 0] = -1          # an unused slot
    scores = _scores(ids.shape, seed=n + 1)
    q_lens = [int(x) for x in rng.integers(0, 200, size=n_q)]
    qp = _qpages(dtype, pages)
    for k in sorted({1, min(10, n), n}):
        got = run_mmr(idx, ids, scores, q_lens, k, 0.5)
        check_picks(ids, scores, q_lens, k, 0.5, got, len(pages))
        slots = None if n <= 100 else [int(x) for x in rng.choice(n, size=40, replace=False)]
        if k <= 10:
            check_sims(KIND[dtype], ids, got, qp, idx.score_scale, slots)


def _nonfinite_pages(seed=3):
    """Unit rows plus rows holding +inf, -inf and NaN, a page of NaN rows only and a page mixing +inf with -inf rows."""
    rng = np.random.default_rng(seed)
    pages = [_unit(rng, n) for n in (40, 64, 65, 3)]
    p = _unit(rng, 33)
    p[5, 0] = np.inf
    pages.append(p)
    p = _unit(rng, 70)
    p[64, 3] = -np.inf
    p[10] = np.nan
    pages.append(p)
    pages.append(np.full((5, 128), np.nan, np.float32))
    p = _unit(rng, 20)
    p[0, 7], p[1, 7] = np.inf, -np.inf
    pages.append(p)
    p = _unit(rng, 2)
    p[:, :] = np.inf
    pages.append(p)
    return pages


@pytest.mark.parametrize("tier", ["hbm", "host"])
@pytest.mark.parametrize("dtype", ["bf16", "fp8"])
def test_non_finite_pages(dtype, tier):
    pages = _nonfinite_pages()
    idx = _index(dtype, tier, pages=pages, key="nonfinite")
    n = len(pages)
    ids = np.array([list(range(n)) + [-1, 2], list(range(n - 1, -1, -1)) + [0, n]], np.int64)
    scores = _scores(ids.shape, seed=9)
    q_lens = [12, 3]
    for lam in (0.5, 0.0, 0.9):
        got = run_mmr(idx, ids, scores, q_lens, ids.shape[1], lam)
        check_picks(ids, scores, q_lens, ids.shape[1], lam, got, n)
        check_sims(KIND[dtype], ids, got, _qpages(dtype, pages), idx.score_scale)
    assert (np.isnan(got[3]) | np.isposinf(got[3])).any()  # non-finite sims do occur


def _flat(idx, queries, ids):
    """The rerank's ranking of each query's list: (ids, scores, counts) on the host."""
    src = torch.from_numpy(np.concatenate(queries)).to(DEV)
    ts, ti, tc = idx.rerank_batch(src, [len(q) for q in queries], torch.from_numpy(ids).to(DEV), ids.shape[1])
    torch.cuda.synchronize()
    return ti.cpu().numpy(), ts.cpu().numpy(), tc.cpu().numpy()


@pytest.mark.parametrize("case", ["bf16", "int8", "fp8", "binary", "bf16_inf", "fp8_nonfinite"])
def test_lambda_one_is_the_flat_ranking(case):
    dtype = case.split("_")[0]
    pages = _nonfinite_pages() if "_" in case else None
    idx = _index(dtype, pages=pages, key="nonfinite" if pages is not None else None)
    n = idx.n_pages
    rng = np.random.default_rng(4)
    queries = [_unit(rng, 9), _unit(rng, 1)]
    if pages is not None:  # tokens that meet the infinities: +inf / -inf / NaN page scores
        queries[0][0] = np.eye(128, dtype=np.float32)[0]
        queries[0][1] = np.eye(128, dtype=np.float32)[7]
    lists = np.array([rng.permutation(n), rng.permutation(n)], np.int64)
    ti, ts, tc = _flat(idx, queries, lists)
    if pages is not None:
        assert not np.isfinite(ts[:, :int(tc.min())]).all()
    q_lens = [len(q) for q in queries]
    for with_sims in (False, True):
        gi, gs, gc, _ = run_mmr(idx, ti, ts, q_lens, ti.shape[1], 1.0, with_sims=with_sims)
        assert np.array_equal(gc, tc)
        assert np.array_equal(gi, ti), (gi, ti)
        assert np.array_equal(gs.view(np.uint32), ts.view(np.uint32))


def test_int8_row_sums_pass_int32():
    plus = np.ones((1100, 128), np.float32)
    pages = [plus, -plus, plus.copy(), plus[:1041]]
    idx = _index("int8", pages=pages, key="overflow")
    ids = np.array([[0, 1, 2, 3]], np.int64)
    got = run_mmr(idx, ids, np.array([[4.0, 3.0, 2.0, 1.0]], np.float32), [1], 4, 0.5)
    s = idx.score_scale
    row = 127 * 127 * 128
    assert 1041 * row > 2 ** 31 - 1

    def sim(S, L):
        return np.float32(np.float32(S) * np.float32(s)) / np.float32(L)

    want = {1: sim(-1100 * row, 1100), 2: sim(1100 * row, 1100), 3: sim(1041 * row, 1041)}
    assert got[0][0, 0] == 0
    for j, w in want.items():
        assert got[3][0, 0, j] == w, (j, got[3][0, 0, j], w)
    check_sims("int8", ids, got, _qpages("int8", pages), s)


def _raw(idx, ids, scores, q_lens, n_q, n_cand, k, lam, scale=None, null=None, stream=None):
    out_i = torch.empty((n_q, max(k, 1)), dtype=torch.int64, device=DEV)
    out_s = torch.empty((n_q, max(k, 1)), dtype=torch.float32, device=DEV)
    out_c = torch.empty((n_q,), dtype=torch.int32, device=DEV)
    args = dict(ids=ctypes.c_void_p(ids.data_ptr()), scores=ctypes.c_void_p(scores.data_ptr()), q_lens=nat.i32_array(q_lens),
                out_i=ctypes.c_void_p(out_i.data_ptr()), out_s=ctypes.c_void_p(out_s.data_ptr()),
                out_c=ctypes.c_void_p(out_c.data_ptr()))
    if null:
        args[null] = None
    return nat.lib.b200ms_mmr_device(idx.h.ptr, args["ids"], args["scores"], n_cand, args["q_lens"], n_q, k,
                                     ctypes.c_float(lam), ctypes.c_float(idx.score_scale if scale is None else scale),
                                     args["out_i"], args["out_s"], args["out_c"], None,
                                     ctypes.c_void_p(torch.cuda.current_stream().cuda_stream if stream is None else stream))


def test_refused_calls_launch_nothing():
    idx = _index("bf16")
    ids = torch.from_numpy(_lists(1, seed=1)).to(DEV)
    sc = torch.from_numpy(_scores(tuple(ids.shape), seed=2)).to(DEV)
    n = int(ids.shape[1])
    assert _raw(idx, ids, sc, [5], 1, n, 3, 0.5) == 0
    torch.cuda.synchronize()
    bad = [dict(null="ids"), dict(null="scores"), dict(null="q_lens"), dict(null="out_i"), dict(null="out_s"),
           dict(null="out_c"), dict(lam=float("nan")), dict(lam=1.5), dict(lam=-0.1), dict(k=0),
           dict(n_cand=0), dict(n_cand=4097), dict(scale=0.0), dict(scale=float("inf")), dict(q_lens=[-1]), dict(n_q=0),
           dict(n_q=1 << 20, n_cand=1024)]
    for b in bad:
        before = idx.launch_count()
        kw = dict(q_lens=[5], n_q=1, n_cand=n, k=3, lam=0.5)
        kw.update(b)
        rc = _raw(idx, ids, sc, kw["q_lens"], kw["n_q"], kw["n_cand"], kw["k"], kw["lam"], scale=b.get("scale"),
                  null=b.get("null"))
        assert rc == -1, (b, rc)
        assert idx.launch_count() == before, b
    # k past every list is not refused: count = the list's distinct valid pages, the rest of the row unused
    big_k = 5000
    out_i = torch.empty((1, big_k), dtype=torch.int64, device=DEV)
    out_s = torch.empty((1, big_k), dtype=torch.float32, device=DEV)
    out_c = torch.empty((1,), dtype=torch.int32, device=DEV)
    assert nat.lib.b200ms_mmr_device(idx.h.ptr, ctypes.c_void_p(ids.data_ptr()), ctypes.c_void_p(sc.data_ptr()), n,
                                     nat.i32_array([5]), 1, big_k, ctypes.c_float(0.5), ctypes.c_float(1.0),
                                     ctypes.c_void_p(out_i.data_ptr()), ctypes.c_void_p(out_s.data_ptr()),
                                     ctypes.c_void_p(out_c.data_ptr()), None,
                                     ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)) == 0
    torch.cuda.synchronize()
    n_valid = int(valid_slots(ids[0].cpu().numpy(), N_PAGES).sum())
    assert int(out_c[0]) == n_valid and (out_i[0, n_valid:] == -1).all() and (out_i[0, :n_valid] >= 0).all()
    empty = MaxSimIndex(dtype="bf16")  # no corpus attached
    before = empty.launch_count()
    assert _raw(empty, ids, sc, [5], 1, n, 3, 0.5) == -3
    assert empty.launch_count() == before
    # host tier: unique candidate pages that need two gather rounds
    host = MaxSimIndex(dtype="bf16", tier="host")
    host.add_pages(PAGES)
    host._attach()
    host.set_option("host_stage_bytes", 1)  # one round holds the largest page, nothing more
    before = host.launch_count()
    rc = _raw(host, ids, sc, [5], 1, n, 3, 0.5)
    assert rc == -1 and host.launch_count() == before
    assert "gather round" in nat.lib.b200ms_last_error(host.h.ptr).decode()
    host.set_option("host_stage_bytes", 2 << 30)  # the default: the same call fits one round
    assert _raw(host, ids, sc, [5], 1, n, 3, 0.5) == 0 and host.launch_count() > before
    torch.cuda.synchronize()


@pytest.mark.parametrize("dtype", ["bf16", "binary"])
def test_ties_go_to_the_lower_slot(dtype):
    """Equal values pick the lower SLOT, not the lower page id: lists in descending id order, equal scores, and two pairs of
    identical pages (equal sims)."""
    idx = _index(dtype)
    ids = np.array([list(range(N_PAGES - 1, -1, -1))], np.int64)
    for scores in (np.ones(ids.shape, np.float32), np.zeros(ids.shape, np.float32), -np.zeros(ids.shape, np.float32)):
        for lam in (1.0, 0.5, 0.0):
            got = run_mmr(idx, ids, scores, [4], ids.shape[1], lam)
            check_picks(ids, scores, [4], ids.shape[1], lam, got, N_PAGES)
            if lam == 1.0:
                assert got[0][0].tolist() == ids[0].tolist()


@pytest.mark.parametrize("dtype", DTYPES)
def test_identical_calls_are_bit_identical(dtype):
    idx = _index(dtype)
    ids = _lists(2, seed=21)
    scores = _scores(ids.shape, seed=22)
    a = run_mmr(idx, ids, scores, [33, 64], 12, 0.4)
    b = run_mmr(idx, ids, scores, [33, 64], 12, 0.4)
    for x, y in zip(a, b):
        assert np.array_equal(x.view(np.uint8), y.view(np.uint8))


STREAM_PAGES = 400


@pytest.mark.parametrize("tier", ["hbm", "host"])
def test_cross_stream_order(tier):
    """One handle, two streams: a long MMR call (400 candidates of 1024 rows, 30 picks, sims) in flight on s1 while a scoring
    call and a second MMR call of the same index run on s2.  The two MMR calls share the handle's pick state and partials
    (and, on the host tier, its staging block); each result must equal its solo run bit for bit."""
    rng = np.random.default_rng(8)
    pages = [_unit(np.random.default_rng(1000 + s), 1024) for s in range(STREAM_PAGES - 8)]
    pages += [_unit(rng, int(n)) for n in (1, 33, 64, 65, 200, 0, 31, 1030)]
    idx = _index("bf16", tier, pages=pages, key="stream")
    ids_a = torch.from_numpy(np.array([rng.permutation(STREAM_PAGES)], np.int64)).to(DEV)
    sc_a = torch.from_numpy(_scores((1, STREAM_PAGES), seed=1)).to(DEV)
    ids_b = torch.from_numpy(_lists(2, seed=3, n_pages=STREAM_PAGES, n=40)).to(DEV)
    sc_b = torch.from_numpy(_scores(tuple(ids_b.shape), seed=4)).to(DEV)
    q = torch.from_numpy(_unit(rng, 40)).to(DEV)
    cand = torch.from_numpy(np.array([rng.permutation(STREAM_PAGES)[:50]], np.int64)).to(DEV)

    def call_a():
        return idx.mmr(ids_a, sc_a, [9], 30, 0.5, with_sims=True)

    def call_b():
        scored = idx.search_device(q, [40], 5) if tier == "hbm" else idx.rerank_batch(q, [40], cand, 5)
        return scored, idx.mmr(ids_b, sc_b, [40, 1], 9, 0.7, with_sims=True)

    solo_a = call_a()
    solo_b = call_b()
    torch.cuda.synchronize()
    s1, s2 = torch.cuda.Stream(), torch.cuda.Stream()
    s1.wait_stream(torch.cuda.current_stream())
    s2.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s1):
        got_a = call_a()
    with torch.cuda.stream(s2):
        got_b = call_b()
    torch.cuda.synchronize()
    for x, y in zip(got_a, solo_a):
        assert torch.equal(x.view(torch.uint8), y.view(torch.uint8))
    for x, y in zip(list(got_b[0]) + list(got_b[1]), list(solo_b[0]) + list(solo_b[1])):
        assert torch.equal(x.view(torch.uint8), y.view(torch.uint8))


def test_value_is_rounded_per_operation():
    """The pick value is the header's expression with every operation rounded to fp32: lambda, rel and red (one-row 1-bit
    pages, sims exact multiples of 1/128) where the two later slots tie, so the lower slot wins; with a fused multiply-add
    the second would (tests/test_mmr_oracle_cpu.py FMA_TIE)."""
    lam, (rel1, red1), (rel2, red2) = np.float32(0.6369617), (0.040973525, 65), (-0.097062, 34)
    ones = np.ones((1, 128), np.float32)

    def flipped(n):  # 128 - n matching sign bits against `ones`: sim = (128 - n) / 128
        x = ones.copy()
        x[0, :n] = -1
        return x

    pages = [ones, flipped(128 - red1), flipped(128 - red2)]
    idx = _index("binary", pages=pages, key="fma")
    ids = np.array([[0, 1, 2]], np.int64)
    scores = np.array([[10.0, rel1, rel2]], np.float32)
    got = run_mmr(idx, ids, scores, [1], 3, float(lam))
    assert got[3][0, 0, 1] == np.float32(red1 / 128) and got[3][0, 0, 2] == np.float32(red2 / 128)
    assert got[0][0].tolist() == [0, 1, 2]
    check_picks(ids, scores, [1], 3, float(lam), got, 3)


# ---------------------------------------------------------------------------------------------------------------- the store
def _planted(seed=17):
    """A query, 6 near-copies of its best page, 8 pages that answer it less well but differently, 30 unrelated pages."""
    rng = np.random.default_rng(seed)
    q = _unit(rng, 8)
    best = np.concatenate([q, _unit(rng, 32)])
    copies = []
    for _ in range(6):
        c = best + np.float32(0.01) * _unit(rng, 40)
        copies.append(c / np.linalg.norm(c, axis=1, keepdims=True))
    distinct = []
    for _ in range(8):
        d = np.float32(0.8) * q + np.float32(0.6) * _unit(rng, 8)
        d = np.concatenate([d / np.linalg.norm(d, axis=1, keepdims=True), _unit(rng, 32)])
        distinct.append(d)
    other = [_unit(rng, 30) for _ in range(30)]
    chunks = []
    for name, group in (("copy", copies), ("distinct", distinct), ("other", other)):
        for i, e in enumerate(group):
            chunks.append(DocumentChunk(document_id=f"{name}{i}", chunk_number=0, content=f"{name}{i}", embedding=e, metadata={}))
    return q, chunks


@pytest.mark.parametrize("kw", [dict(), dict(fde_candidates=64), dict(sign_candidates=64),
                                dict(sign_candidates=64, corpus_tier="host")], ids=["exhaustive", "fde", "sign", "sign_host"])
def test_store_returns_one_copy_and_four_distinct_pages(kw):
    q, chunks = _planted()
    store = B200MultiVectorStore(mode="bf16", coalesce_queries=False, **kw)
    asyncio.run(store.store_embeddings(chunks))
    flat = asyncio.run(store.query_similar(q, k=5))
    assert [c.document_id[:4] for c in flat] == ["copy"] * 5
    res = asyncio.run(store.query_similar_mmr(q, k=5, fetch_k=20, lambda_mult=0.5))
    docs = [c.document_id for c in res]
    assert len(docs) == 5 and len(set(docs)) == 5
    assert docs[0].startswith("copy") and sum(d.startswith("copy") for d in docs) == 1, docs
    assert all(d.startswith("distinct") for d in docs[1:]), docs
    assert store.last_query_timing["mmr_ms"] > 0
    by_doc = {c.document_id: c.score for c in asyncio.run(store.query_similar(q, k=len(chunks)))}
    assert all(c.score == by_doc[c.document_id] for c in res)  # query_similar's scores
    allowed = ["copy2", "copy4", "other3", "distinct6"]
    res = asyncio.run(store.query_similar_mmr(q, k=5, fetch_k=20, lambda_mult=0.5, doc_ids=allowed))
    assert {c.document_id for c in res} <= set(allowed) and len(res) == 4
    assert res[0].document_id in ("copy2", "copy4")
    assert sum(c.document_id.startswith("copy") for c in res) == 2  # nothing else left to pick
    same = [(c.document_id, c.score) for c in asyncio.run(store.query_similar_mmr(q, k=3, lambda_mult=1.0))]
    assert same == [(c.document_id, c.score) for c in asyncio.run(store.query_similar(q, k=3))]
    store.close()
