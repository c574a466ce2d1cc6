"""b200ms_explain_device / MaxSimIndex.explain / B200MultiVectorStore.explain_chunks on an H100 (run with -m gpu).

For every corpus dtype: token scores, best rows and maps against the numpy oracle (tests/explain_oracle.py) over query lengths
1 .. 1030 and page lengths 0 .. 1030, with unused slots, repeated pages, shared and per-query lists; the kernel's own
consistency (score == map at the best row, the lowest such row, never a padding row); ties; that the token scores add up
to the rerank's page scores; that every output entry is written (0xA5 pre-fill); host tier == HBM tier bit for bit, also
over several staging rounds; refusals; and the store's explain_chunks across deletes, compaction, save/load and replay.
"""
import asyncio
import ctypes

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

torch = pytest.importorskip("torch")
if not torch.cuda.is_available():  # pragma: no cover - the gpu marker normally deselects these on CPU boxes
    pytest.skip("CUDA device required", allow_module_level=True)

from explain_oracle import maxsim_explain_np, quantise  # noqa: E402
from morphik_core_b200 import _native as nat  # noqa: E402
from morphik_core_b200.index import MaxSimIndex  # noqa: E402
from morphik_core_b200.models import DocumentChunk  # noqa: E402
from morphik_core_b200.store import B200MultiVectorStore  # noqa: E402
from oracle import maxsim_oracle as orc  # noqa: E402

DTYPES = {"bf16": "bf16", "int8": "int8", "fp8": "fp8", "binary": "bits"}
QLENS = [1, 31, 32, 33, 128, 129, 1030]
PLENS = [0, 1, 31, 32, 33, 1024, 1030]
FILL = 0xA5
SENTINEL32 = 0xA5A5A5A5
# map tolerance against the float64 oracle on the same rounded inputs: the fp32 sum of 128 products of unit-norm rows (bf16)
# and of rows scaled by 64 (fp8, 64^2 = 4096 times larger)
TOL = {"bf16": 1e-4, "fp8": 4096 * 1e-4}


def _unit(rng, n):
    x = rng.standard_normal((n, 128)).astype(np.float32)
    return x / np.maximum(np.linalg.norm(x, axis=1, keepdims=True), 1e-9)


def _corpus(seed=7):
    """PLENS pages, a tie page (row 5 repeated at 17 and 33), a page of one repeated row, and some random pages."""
    rng = np.random.default_rng(seed)
    pages = [_unit(rng, n) for n in PLENS]
    tie = _unit(rng, 40)
    tie[[17, 33]] = tie[5]
    pages.append(tie)
    pages.append(np.repeat(_unit(rng, 1), 50, axis=0))
    pages += [_unit(rng, int(n)) for n in rng.integers(1, 300, size=5)]
    return pages


PAGES = _corpus()
TIE_PAGE, SAME_PAGE = len(PLENS), len(PLENS) + 1
N_PAGES = len(PAGES)
_INDEXES = {}


def _index(dtype, tier="hbm"):
    key = (dtype, tier)
    if key not in _INDEXES:
        idx = MaxSimIndex(dtype=dtype, tier=tier)
        idx.add_pages(PAGES)
        idx._attach()
        _INDEXES[key] = idx
    return _INDEXES[key]


def _queries(lens, seed):
    rng = np.random.default_rng(seed)
    qs = [_unit(rng, n) for n in lens]
    if lens and lens[0] >= 3:  # tokens aimed at the tie page and the all-equal page
        qs[0][0] = PAGES[TIE_PAGE][5]
        qs[0][1] = PAGES[SAME_PAGE][0]
    return qs


def _ids(n_q, seed):
    """Per-query lists: every PLENS page, the tie pages, -1, an id past the corpus, a repeated page, a random page."""
    rng = np.random.default_rng(seed)
    rows = []
    for _ in range(n_q):
        lst = list(range(len(PLENS))) + [TIE_PAGE, SAME_PAGE, -1, N_PAGES + 3, 4, int(rng.integers(0, N_PAGES))]
        rng.shuffle(lst)
        rows.append(lst)
    return np.asarray(rows, dtype=np.int64)


def explain_raw(idx, queries, ids, map_rows, scale=1.0, sim_map=True):
    """b200ms_explain_device straight through the C-ABI into 0xA5-filled outputs (host numpy results)."""
    lens = [int(q.shape[0]) for q in queries]
    n_q, n_cand, t_max = len(lens), ids.shape[1], max(lens)
    src = torch.from_numpy(np.concatenate(queries)).to(idx.device)
    ids_d = torch.from_numpy(np.ascontiguousarray(ids)).to(idx.device)

    def filled(*shape):
        n = int(np.prod(shape))
        return torch.full((4 * n,), FILL, dtype=torch.uint8, device=idx.device).view(torch.int32).view(*shape)

    ts, br = filled(n_q, n_cand, t_max), filled(n_q, n_cand, t_max)
    sm = filled(n_q, n_cand, t_max, map_rows) if sim_map and map_rows else None
    with torch.cuda.device(idx.device):
        idx.h.check(nat.lib.b200ms_explain_device(
            idx.h.ptr, ctypes.c_void_p(src.data_ptr()), nat.F32, nat.i32_array(lens), n_q, ctypes.c_void_p(ids_d.data_ptr()),
            n_cand, ctypes.c_float(idx.i8_scale), ctypes.c_float(scale), ctypes.c_void_p(ts.data_ptr()),
            ctypes.c_void_p(br.data_ptr()), None if sm is None else ctypes.c_void_p(sm.data_ptr()), int(map_rows),
            ctypes.c_void_p(torch.cuda.current_stream(idx.device).cuda_stream)), "b200ms_explain_device")
    torch.cuda.synchronize(idx.device)
    ts_u, br_i = ts.cpu().numpy().view(np.uint32), br.cpu().numpy()
    sm_u = None if sm is None else sm.cpu().numpy().view(np.uint32)
    for a in (ts_u, br_i.view(np.uint32)) + (() if sm_u is None else (sm_u,)):
        assert not (a == SENTINEL32).any(), "an output entry was left unwritten"
    return ts_u.view(np.float32), br_i, None if sm_u is None else sm_u.view(np.float32)


def _check(dtype, queries, ids, ts, br, sm, map_rows):
    kind = DTYPES[dtype]
    lens = [p.shape[0] for p in PAGES]
    off = orc.page_offsets(lens)
    rows = quantise(np.concatenate(PAGES), kind)
    t_max = max(q.shape[0] for q in queries)
    for qi, q in enumerate(queries):
        T = q.shape[0]
        best, arg, maps = maxsim_explain_np(quantise(q, kind), rows, off, kind)
        # tokens past this query's length
        assert (ts[qi, :, T:] == 0).all() and (br[qi, :, T:] == -1).all()
        if sm is not None:
            assert np.isneginf(sm[qi, :, T:]).all()
        for j, pid in enumerate(ids[qi]):
            t, b = ts[qi, j, :T], br[qi, j, :T]
            if not (0 <= pid < N_PAGES) or lens[pid] == 0:
                assert (t == 0).all() and (b == -1).all(), (dtype, qi, j, pid)
                if sm is not None:
                    assert np.isneginf(sm[qi, j]).all()
                continue
            L = lens[pid]
            assert ((b >= 0) & (b < L)).all(), "a best row outside the page's true rows"
            if kind in ("int8", "bits"):
                assert np.array_equal(t.astype(np.int64), best[pid]), (dtype, qi, pid)
                assert np.array_equal(b, arg[pid]), (dtype, qi, pid)
            else:
                tol = TOL[dtype]
                assert np.abs(t - best[pid]).max() <= tol, (dtype, qi, pid)
                assert np.abs(maps[pid][np.arange(T), b] - best[pid]).max() <= tol  # the oracle's value at the row
            if sm is None:
                continue
            m = sm[qi, j, :T]
            c = min(L, map_rows)
            assert np.isneginf(m[:, c:]).all()
            if kind in ("int8", "bits"):
                assert np.array_equal(m[:, :c].astype(np.int64), maps[pid][:, :c])
            else:
                assert np.abs(m[:, :c] - maps[pid][:, :c]).max() <= TOL[dtype]
            # self-consistency, exact: the score is the map at the best row, the lowest row of the kernel's own max
            cov = np.flatnonzero(b < map_rows)
            assert np.array_equal(m[cov, b[cov]].view(np.uint32), t[cov].view(np.uint32))
            if L <= map_rows:
                own = m[:, :L]
                assert np.array_equal(own.max(axis=1), t)
                assert np.array_equal(own.argmax(axis=1), b)
    assert ts.shape[2] == t_max


@pytest.mark.parametrize("dtype", list(DTYPES))
def test_against_the_oracle(dtype):
    idx = _index(dtype)
    q_short = _queries([q for q in QLENS if q < 1000], seed=1)
    ids = _ids(len(q_short), seed=2)
    ts, br, sm = explain_raw(idx, q_short, ids, map_rows=1100)
    _check(dtype, q_short, ids, ts, br, sm, 1100)
    q_long = _queries([1030, 33], seed=3)
    ids_l = _ids(2, seed=4)
    ts, br, sm = explain_raw(idx, q_long, ids_l, map_rows=40)
    _check(dtype, q_long, ids_l, ts, br, sm, 40)
    # ties: the tie page answers token 0 of query 0 with row 5 (copies at 17 and 33), the all-equal page with row 0
    j_tie = list(ids_l[0]).index(TIE_PAGE)
    j_same = list(ids_l[0]).index(SAME_PAGE)
    assert br[0, j_tie, 0] == 5 and br[0, j_same, 1] == 0
    assert (br[0, j_same, :1030] == 0).all()


@pytest.mark.parametrize("dtype", list(DTYPES))
def test_shared_list_and_python_api(dtype):
    idx = _index(dtype)
    qs = _queries([40, 7, 130], seed=5)
    shared = np.asarray([3, -1, 5, TIE_PAGE, 3, 99], dtype=np.int64)
    ts, br, sm = idx.explain(qs, shared, map_rows=64)
    ts_r, br_r, sm_r = explain_raw(idx, qs, np.repeat(shared[None], 3, axis=0), 64, scale=idx.score_scale)
    assert np.array_equal(ts.cpu().numpy().view(np.uint32), ts_r.view(np.uint32))
    assert np.array_equal(br.cpu().numpy(), br_r)
    assert np.array_equal(sm.cpu().numpy().view(np.uint32), sm_r.view(np.uint32))
    ts2, br2, sm2 = idx.explain([torch.from_numpy(q).to(idx.device) for q in qs], torch.from_numpy(shared))
    assert sm2 is None and torch.equal(ts2, ts) and torch.equal(br2, br)


DEVIATION = {}


@pytest.mark.parametrize("dtype", list(DTYPES))
def test_adds_up_to_the_rerank(dtype):
    idx = _index(dtype)
    qs = _queries([1, 33, 129, 1030], seed=6)
    ids = _ids(len(qs), seed=7)
    raw, _, _ = explain_raw(idx, qs, ids, 0, sim_map=False)
    src = torch.from_numpy(np.concatenate(qs)).to(idx.device)
    n_cand = ids.shape[1]
    rs, ri, rc = idx.rerank_batch(src, [q.shape[0] for q in qs], torch.from_numpy(ids).to(idx.device), n_cand)
    rs, ri, rc = rs.cpu().numpy(), ri.cpu().numpy(), rc.cpu().numpy()
    s = np.float32(idx.score_scale)
    worst = 0.0
    for qi in range(len(qs)):
        got = {int(p): float(v) for p, v in zip(ri[qi, :rc[qi]], rs[qi, :rc[qi]])}
        for j, pid in enumerate(ids[qi]):
            if not (0 <= pid < N_PAGES):
                continue
            if dtype in ("int8", "binary"):
                total = raw[qi, j].astype(np.int64).sum()
                assert np.float32(np.float32(total) * s) == np.float32(got.get(pid, 0.0)), (dtype, qi, pid)
            else:
                total = raw[qi, j].astype(np.float64).sum() * float(s)
                want = got.get(pid, 0.0)
                dev = abs(total - want) / max(abs(want), 1e-30)
                worst = max(worst, dev)
                assert dev <= 2e-6, (dtype, qi, pid, total, want)
    DEVIATION[dtype] = worst
    print(f"[explain] {dtype}: largest relative deviation of sum_t token_scores from the rerank score: {worst:.3g}")


@pytest.mark.parametrize("dtype", list(DTYPES))
def test_host_tier_is_bit_identical(dtype):
    hbm, host = _index(dtype), _index(dtype, "host")
    qs = _queries([33, 1030, 5], seed=8)
    ids = _ids(len(qs), seed=9)
    want = explain_raw(hbm, qs, ids, 48)
    uniq = len({int(p) for p in ids.reshape(-1) if 0 <= p < N_PAGES})
    for stage in (0, 1):
        if stage:
            host.set_option("host_stage_bytes", 1)  # raised to the largest page: about one page per round
        got = explain_raw(host, qs, ids, 48)
        for a, b in zip(want, got):
            assert np.array_equal(a.view(np.uint32), b.view(np.uint32))
        st = host.gather_stats()
        assert st["unique_pages"] == uniq
        assert (st["rounds"] > 1) == bool(stage)
    host.set_option("host_stage_bytes", 2 << 30)
    only_empty = np.asarray([[0, -1, 0]], dtype=np.int64)  # nothing to gather: every slot is a fill
    a = explain_raw(hbm, qs[:1], only_empty, 8)
    b = explain_raw(host, qs[:1], only_empty, 8)
    for x, y in zip(a, b):
        assert np.array_equal(x.view(np.uint32), y.view(np.uint32))
    assert host.gather_stats()["rounds"] == 0


def test_refusals():
    h = nat.Handle(0)
    q = torch.zeros((4, 128), dtype=torch.float32, device="cuda")
    ids = torch.zeros((1, 4), dtype=torch.int64, device="cuda")
    out = torch.empty(64, dtype=torch.float32, device="cuda")
    vp = lambda t: ctypes.c_void_p(t.data_ptr())  # noqa: E731
    lens = nat.i32_array([4])

    def call(hp=h.ptr, qp=vp(q), dt=nat.F32, ql=lens, n_q=1, ip=vp(ids), n_cand=4, ts=vp(out), br=vp(out), mr=0, sm=None):
        return nat.lib.b200ms_explain_device(hp, qp, dt, ql, n_q, ip, n_cand, ctypes.c_float(1), ctypes.c_float(1), ts, br, sm,
                                             mr, None)

    assert call() == -3  # no corpus
    assert call(hp=None) == -1
    assert call(qp=None) == -1 and call(ql=None) == -1 and call(ip=None) == -1 and call(ts=None) == -1 and call(br=None) == -1
    assert call(dt=nat.I8) == -1 and call(dt=99) == -1
    assert call(mr=-1) == -1
    assert call(n_q=0) == -1 and call(n_cand=0) == -1
    assert call(n_cand=1 << 30) == -1
    assert call(n_q=2, ql=nat.i32_array([4, 4]), n_cand=1 << 29) == -1  # n_q * n_cand = 2^30
    assert call(ql=nat.i32_array([-1])) == -1
    h.close()


def _run(coro):
    return asyncio.run(coro)


def _chunks(rng, n_docs=6, per_doc=3):
    out = []
    for d in range(n_docs):
        for c in range(per_doc):
            out.append(DocumentChunk(document_id=f"doc{d}", content=f"{d}-{c}", chunk_number=c, metadata={},
                                     embedding=_unit(rng, int(rng.integers(20, 200)))))
    return out


def _assert_store_explains(store, q, ids_visible, dtype):
    hits = _run(store.query_similar_batch([q], k=len(store.catalog)))[0]
    score_of = {(h.document_id, h.chunk_number): h.score for h in hits}
    recs = _run(store.explain_chunks(q, ids_visible + ids_visible[:1] + [("nope", 0)], with_map=True))
    assert [(r["document_id"], r["chunk_number"]) for r in recs] == [k for k in ids_visible if k in score_of]
    for r in recs:
        want = score_of[(r["document_id"], r["chunk_number"])]
        assert abs(r["score"] - want) <= 2e-6 * max(abs(want), 1.0), (dtype, r["score"], want)
        n_rows = r["sim_map"].shape[1]
        assert r["token_scores"].shape == (q.shape[0],) and ((r["best_patch"] >= 0) & (r["best_patch"] < n_rows)).all()
        assert np.array_equal(r["sim_map"][np.arange(q.shape[0]), r["best_patch"]], r["token_scores"])
    return {(r["document_id"], r["chunk_number"]): (r["token_scores"], r["best_patch"]) for r in recs}


@pytest.mark.parametrize("dtype", ["bf16", "int8", "fp8", "binary"])
def test_store_explain_chunks(dtype, tmp_path):
    rng = np.random.default_rng(11)
    store = B200MultiVectorStore(mode=dtype, compact_dead_fraction=0.0, coalesce_queries=False)
    chunks = _chunks(rng)
    _run(store.store_embeddings(chunks[:9], app_id="a"))
    _run(store.store_embeddings(chunks[9:], app_id="b"))
    q = _unit(rng, 20)
    keys = [("doc4", 1), ("doc1", 0), ("doc5", 2), ("doc2", 2)]
    before = _assert_store_explains(store, q, keys, dtype)
    # app_id visibility as get_chunks_by_id: doc0..2 are app "a", doc3..5 app "b"
    vis = [(c.document_id, c.chunk_number) for c in _run(store.get_chunks_by_id(keys, app_id="a"))]
    assert [(r["document_id"], r["chunk_number"]) for r in _run(store.explain_chunks(q, keys, app_id="a"))] == vis == [
        ("doc1", 0), ("doc2", 2)]
    # delete another document (compaction moves every later page id), save/load
    _run(store.delete_chunks_by_document_id("doc3"))
    after = _assert_store_explains(store, q, keys, dtype)
    for k in keys:
        assert np.array_equal(before[k][0], after[k][0]) and np.array_equal(before[k][1], after[k][1])
    store.save(str(tmp_path / "ck"))
    loaded = B200MultiVectorStore.load(str(tmp_path / "ck"), coalesce_queries=False)
    again = _assert_store_explains(loaded, q, keys, dtype)
    for k in keys:
        assert np.array_equal(before[k][0], again[k][0]) and np.array_equal(before[k][1], again[k][1])
    loaded.close()
    store.close()
    # journal replay
    durable = B200MultiVectorStore.open(str(tmp_path / "j"), mode=dtype, coalesce_queries=False)
    _run(durable.store_embeddings(chunks[:9], app_id="a"))
    _run(durable.store_embeddings(chunks[9:], app_id="b"))
    _run(durable.delete_chunks_by_document_id("doc3"))
    durable.close()
    replayed = B200MultiVectorStore.open(str(tmp_path / "j"), mode=dtype, coalesce_queries=False)
    again = _assert_store_explains(replayed, q, keys, dtype)
    for k in keys:
        assert np.array_equal(before[k][0], again[k][0]) and np.array_equal(before[k][1], again[k][1])
    replayed.close()
