"""b200ms_pair_maxsim_device / b200ms_duplicate_groups_device and the store's duplicate calls on an H100 (run with -m gpu).

sim(a -> b) against b200ms_mmr_device's sim for the same pair bit for bit on every dtype, sim(b -> a) against MMR with the
roles swapped (bit for bit on int8 and bits, within oracle.scoring.TOL of the float64 oracle on bf16 and fp8), over page
lengths 0 .. 1030 and a page long enough for the global column scratch, self-pairs and repeated pairs; rows holding
+-inf, NaN and +-0 (MMR's NaN rule) and int8 rows at -128 / 127 whose sums pass int32, both directions against MMR; pairs of
pages past 4 GiB of corpus against the float64 reference of tests/scale_reference.py; the components against union-find on
random graphs, a 100 000-page path in worst order, a star, no edges and masked pages; the store end to end on a planted
corpus (the exhaustive pair set against the oracle's top n_candidates, doc_ids and app_id filters); and each export in
flight on one stream while another call of the handle runs on a second."""
import asyncio
import gc

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

torch = pytest.importorskip("torch")
if not torch.cuda.is_available():  # pragma: no cover - the gpu marker normally deselects these on CPU boxes
    pytest.skip("CUDA device required", allow_module_level=True)

from duplicates_oracle import canonical_pairs, collapsed_topk, edges, pair_sims, union_find_labels  # noqa: E402
from mmr_oracle import page_sum, quantise_rows  # noqa: E402
from morphik_core_b200.index import MaxSimIndex  # noqa: E402
from morphik_core_b200.models import DocumentChunk  # noqa: E402
from morphik_core_b200.store import B200MultiVectorStore  # noqa: E402
from oracle.scoring import TOL, i32_reported  # noqa: E402

KIND = {"bf16": "bf16", "int8": "int8", "fp8": "fp8", "binary": "bits"}
DTYPES = list(KIND)
PLENS = [0, 1, 31, 32, 33, 63, 64, 65, 127, 128, 129, 1024, 1030, 2100]  # 2100 rows: columns in global scratch
DEV = torch.device("cuda", 0)
BIT_IDENTICAL = {}  # float dtypes: pairs whose sim(b -> a) equals MMR's swapped value bit for bit (printed with -s)


def _unit(rng, n):
    x = rng.standard_normal((n, 128)).astype(np.float32)
    return x / np.maximum(np.linalg.norm(x, axis=1, keepdims=True), 1e-9)


def _pages(seed=5):
    rng = np.random.default_rng(seed)
    pages = [_unit(rng, n) for n in PLENS]
    near = pages[PLENS.index(65)] + np.float32(0.05) * _unit(rng, 65)
    pages.append(near / np.linalg.norm(near, axis=1, keepdims=True))
    pages.append(pages[PLENS.index(129)][::2].copy())  # a subset of another page's rows
    return pages


PAGES = _pages()
_INDEXES = {}


def _index(dtype):
    if dtype not in _INDEXES:
        idx = MaxSimIndex(dtype=dtype)
        idx.add_pages(PAGES)
        idx._attach()
        _INDEXES[dtype] = idx
    return _INDEXES[dtype]


def _dev(x, dt=torch.int64):
    return torch.as_tensor(np.ascontiguousarray(x), dtype=dt).to(DEV)


def _pairs():
    n = len(PAGES)
    a, b = np.meshgrid(np.arange(n), np.arange(n), indexing="ij")
    a, b = a.ravel(), b.ravel()
    return np.concatenate([a, [3, 3]]), np.concatenate([b, [12, 12]])  # every ordered pair, self-pairs, a repeat


def _mmr_sim(idx, src, dst):
    """MMR's sim(src[i] -> dst[i]) for each pair with src != dst: list [dst, src], dst picked first."""
    ids = np.stack([dst, src], axis=1).astype(np.int64)
    scores = np.tile(np.array([1.0, 0.0], np.float32), (len(src), 1))
    _, _, _, sims = idx.mmr(_dev(ids), _dev(scores, torch.float32), [1] * len(src), 1, 0.5, with_sims=True)
    return sims[:, 0, 1].cpu().numpy()


@pytest.mark.parametrize("b1_tensor", [0, 1])
@pytest.mark.parametrize("dtype", DTYPES)
def test_pair_sims_match_mmr_and_the_oracle(dtype, b1_tensor):
    if dtype != "binary" and b1_tensor == 1:
        pytest.skip("b1_tensor only selects the 1-bit scan")
    idx = _index(dtype)
    idx.set_option("b1_tensor", b1_tensor)
    a, b = _pairs()
    sab, sba = idx.pair_maxsim(_dev(a), _dev(b))
    torch.cuda.synchronize()
    sab, sba = sab.cpu().numpy(), sba.cpu().numpy()
    distinct = a != b
    m_ab = _mmr_sim(idx, a[distinct], b[distinct])
    m_ba = _mmr_sim(idx, b[distinct], a[distinct])
    assert np.array_equal(sab[distinct].view(np.uint32), m_ab.view(np.uint32))
    kind = KIND[dtype]
    exact = kind in ("int8", "bits")
    if exact:
        assert np.array_equal(sba[distinct].view(np.uint32), m_ba.view(np.uint32))
    else:
        BIT_IDENTICAL[dtype] = (int(np.sum(sba[distinct].view(np.uint32) == m_ba.view(np.uint32))), int(distinct.sum()))
        print(f"{dtype}: sim(b -> a) bit-identical to MMR's on {BIT_IDENTICAL[dtype][0]} of {BIT_IDENTICAL[dtype][1]} pairs")
    qp = [quantise_rows(p, kind) for p in PAGES]
    w_ab, w_ba = pair_sims(qp, a, b, kind, idx.score_scale)
    for got, want in ((sab, w_ab), (sba, w_ba)):
        if exact:
            assert np.array_equal(got, want.astype(np.float32))
        else:
            assert np.all(np.abs(got - want) <= TOL[dtype] * np.maximum(np.abs(want), 1.0))
    # a page without rows is 0 both ways; repeated pairs repeat their values
    empty = (a == 0) | (b == 0)
    assert np.all(sab[empty] == 0) and np.all(sba[empty] == 0)
    assert sab[-1] == sab[-2] and sba[-1] == sba[-2]


def test_ids_outside_the_corpus_give_nan():
    idx = _index("int8")
    sab, sba = idx.pair_maxsim(_dev([-1, 1, len(PAGES)]), _dev([1, 1000, 2]))
    torch.cuda.synchronize()
    assert np.all(np.isnan(sab.cpu().numpy())) and np.all(np.isnan(sba.cpu().numpy()))


def _same(got, want):
    """Bit for bit, a NaN matching any NaN (the NaN rule, not the payload)."""
    got, want = np.asarray(got, np.float32), np.asarray(want, np.float32)
    return bool(np.all((got.view(np.uint32) == want.view(np.uint32)) | (np.isnan(got) & np.isnan(want))))


def _check_against_mmr(idx, n_pages, what):
    a, b = np.meshgrid(np.arange(n_pages), np.arange(n_pages), indexing="ij")
    a, b = a.ravel(), b.ravel()
    a, b = a[a != b], b[a != b]
    sab, sba = idx.pair_maxsim(_dev(a), _dev(b))
    torch.cuda.synchronize()
    sab, sba = sab.cpu().numpy(), sba.cpu().numpy()
    assert np.array_equal(sab.view(np.uint32), _mmr_sim(idx, a, b).view(np.uint32)), what
    assert _same(sba, _mmr_sim(idx, b, a)), what
    return a, b, sab, sba


SPECIALS = [1.0, 2.0, -3.0, np.inf, -np.inf, np.nan, 0.0, -0.0, 0.5]
# per-page palettes, so that some pairs sum to finite values, some to +-inf and some to NaN
PALETTES = [[1.0, 2.0, -3.0, 0.5, 0.0, -0.0], [1.0, 2.0, 0.5, np.inf], [1.0, -3.0, 0.5, -np.inf, -0.0],
            [1.0, 2.0, 0.5, np.nan], SPECIALS]


@pytest.mark.parametrize("dtype", DTYPES)
def test_inf_nan_and_signed_zero_rows(dtype):
    """Rows with one nonzero element drawn from a page's palette of SPECIALS: every product is exact, so both directions equal MMR's value
    whatever order the maxima and sums take (NaN rows, 0 * inf NaNs, -0 rows and all-NaN pages included)."""
    rng = np.random.default_rng(9)
    div = 64.0 if dtype == "fp8" else 1.0
    pages = []
    for p in range(15):
        palette = PALETTES[p % len(PALETTES)]
        rows = np.zeros((int(rng.integers(1, 140)), 128), np.float32)
        for r in range(len(rows)):
            rows[r, int(rng.integers(0, 4))] = palette[int(rng.integers(0, len(palette)))] / div
        pages.append(rows)
    pages.append(np.full((3, 128), np.nan, np.float32))
    pages.append(np.full((2, 128), -0.0, np.float32))
    idx = MaxSimIndex(dtype=dtype)
    try:
        idx.add_pages(pages)
        idx._attach()
        _, _, sab, sba = _check_against_mmr(idx, len(pages), dtype)
        if dtype in ("bf16", "fp8"):  # the crafted values reach the sums
            assert np.isnan(sab).any() and (np.isfinite(sab) & (sab != 0)).any()
        if dtype == "bf16":
            assert np.isinf(sab).any() and np.isinf(sba).any()
    finally:
        idx.close()


def _pad32(rows, lens):
    out, o = [], 0
    for n in lens:
        page = rows[o:o + n]
        o += n
        if n:
            out.append(np.concatenate([page, np.repeat(page[-1:], -n % 32, axis=0)]))
    return np.concatenate(out)


def test_int8_rows_at_the_integer_limits():
    """-128 / +-127 codes: a row pair scores up to 2^21, so 1100-row pages pass int32 in both directions; exact against MMR
    and the int64 oracle."""
    full = lambda v, n: np.full((n, 128), v, np.int8)  # noqa: E731
    alt = np.where(np.arange(128) % 2, -127, 127).astype(np.int8)
    pages = [full(-128, 1100), np.concatenate([full(127, 550), full(-127, 550)]), full(-128, 1), np.tile(alt, (65, 1)),
             full(127, 33), np.concatenate([full(-128, 40), full(127, 40)]), full(127, 1100), np.zeros((0, 128), np.int8)]
    lens = [len(p) for p in pages]
    idx = MaxSimIndex(dtype="int8")
    try:
        idx.append_packed(torch.from_numpy(np.ascontiguousarray(_pad32(np.concatenate(pages).view(np.uint8), lens))).to(DEV),
                          lens)
        idx._attach()
        a, b, sab, sba = _check_against_mmr(idx, len(pages), "int8 limits")
        w_ab, w_ba = pair_sims(pages, a, b, "int8", idx.score_scale)
        assert np.array_equal(sab.view(np.uint32), w_ab.view(np.uint32))
        assert np.array_equal(sba.view(np.uint32), w_ba.view(np.uint32))
        assert page_sum(pages[0], pages[2], "int8") > 2**31 and page_sum(pages[6], pages[0], "int8") < -(2**31)
    finally:
        idx.close()


SCALE_PAGES = {"bf16": 20480, "int8": 40960}  # tests/scale_reference.py corpora past 4 GiB (test_gpu_page_query_scale.py)
FOUR_GIB = 1 << 32


@pytest.mark.parametrize("dtype", list(SCALE_PAGES))
def test_pairs_past_4gib(dtype):
    import page_query_oracle as pqo
    import scale_reference as sr

    rows = int(sr.padded_rows(sr.page_lens(SCALE_PAGES[dtype], 0)).sum())
    gc.collect()
    torch.cuda.empty_cache()
    free, _ = torch.cuda.mem_get_info(DEV)
    need = rows * sr.ROW_BYTES[dtype] + (4 << 30)
    if free < need:
        pytest.skip(f"the {dtype} corpus needs {need / 2**30:.1f} GiB of device memory, {free / 2**30:.1f} GiB are free")
    idx = sr.build(dtype, SCALE_PAGES[dtype], 0)
    try:
        lens = np.asarray(idx.page_lens, np.int64)
        starts = pqo.starts_of(lens)
        live = np.flatnonzero(lens > 0)
        past = np.flatnonzero((starts[:-1] * idx.row_bytes >= FOUR_GIB) & (lens > 0))
        assert len(past) > 100
        rng = np.random.default_rng(4)
        sel = np.unique(np.concatenate([rng.choice(past, 40, replace=False), live[[0, -1]]]))
        packed = idx.packed_rows()
        sub = torch.cat([packed[starts[p]:starts[p] + (lens[p] + 31) // 32 * 32] for p in sel])
        ref = pqo.page_query_reference(dtype, sub, lens[sel], list(range(len(sel))))  # [j, s] = sim(sel j -> sel s)
        ai = rng.integers(0, len(sel), 300)
        bi = rng.integers(0, len(sel), 300)
        sab, sba = idx.pair_maxsim(_dev(sel[ai]), _dev(sel[bi]))
        torch.cuda.synchronize()
        sab, sba = sab.cpu().numpy(), sba.cpu().numpy()
        for got, src, dst in ((sab, ai, bi), (sba, bi, ai)):
            want = ref[src, dst]
            if dtype == "int8":
                n = lens[sel[src]]
                sums = np.rint(want * n * sr._score_divisor(dtype)).astype(np.int64)
                exact = i32_reported(sums, idx.score_scale) / n.astype(np.float32)
                assert np.array_equal(got.view(np.uint32), exact.astype(np.float32).view(np.uint32))
            else:
                assert np.all(np.abs(got - want) <= TOL[dtype] * np.maximum(np.abs(want), 1e-3))
    finally:
        idx.close()
        del idx
        gc.collect()
        torch.cuda.empty_cache()


_LABEL_INDEX = {}


def _label_index(n):
    """A 1-bit corpus of n one-row pages: duplicate_groups only needs the page count."""
    if n not in _LABEL_INDEX:
        idx = MaxSimIndex(dtype="binary")
        idx.add_pages([np.ones((1, 128), np.float32)] * n)
        idx._attach()
        _LABEL_INDEX[n] = idx
    return _LABEL_INDEX[n]


def _groups(idx, a, b, sab, sba, t, allowed=None):
    mask = None
    if allowed is not None:
        from morphik_core_b200.catalog import PageCatalog

        mask = _dev(PageCatalog.mask_words(np.asarray(allowed, bool)).view(np.int32), torch.int32)
    lab = idx.duplicate_groups(_dev(a), _dev(b), _dev(sab, torch.float32), _dev(sba, torch.float32), t, mask)
    torch.cuda.synchronize()
    return lab.cpu().numpy()


@pytest.mark.parametrize("seed", range(4))
def test_components_match_union_find(seed):
    rng = np.random.default_rng(seed)
    n = 3000
    idx = _label_index(n)
    m = 4000
    a, b = rng.integers(0, n, m), rng.integers(0, n, m)
    a[:50] = b[:50]  # self-pairs
    sab, sba = rng.random(m).astype(np.float32), rng.random(m).astype(np.float32)
    sab[50:80] = np.nan
    allowed = rng.random(n) > 0.1 if seed % 2 else None
    for t in (0.3, 0.7):
        want = union_find_labels(n, edges(a, b, sab, sba, t, allowed), allowed)
        assert np.array_equal(_groups(idx, a, b, sab, sba, t, allowed), want)


@pytest.mark.parametrize("order", ["descending", "interleaved"])
def test_long_path_in_worst_order(order):
    n = 100_000
    idx = _label_index(n)
    # the path 0 - 1 - ... - n-1: edges from its far end first, or every other edge first, each edge's larger page first
    e = np.arange(n - 1)[::-1] if order == "descending" else np.concatenate([np.arange(0, n - 1, 2), np.arange(1, n - 1, 2)])
    a, b = e + 1, e
    s = np.ones(n - 1, np.float32)
    assert np.array_equal(_groups(idx, a, b, s, s, 0.5), np.zeros(n, np.int64))
    allowed = np.ones(n, bool)
    allowed[n // 2] = False  # a hidden page cuts the path: nothing joins through it
    want = np.where(np.arange(n) < n // 2, 0, n // 2 + 1)
    want[n // 2] = -1
    assert np.array_equal(_groups(idx, a, b, s, s, 0.5, allowed), want)


def test_star_and_no_edges():
    n = 5000
    idx = _label_index(n)
    leaves = np.arange(n - 1)
    a, b = np.full(n - 1, n - 1), np.roll(leaves, 7)
    s = np.ones(n - 1, np.float32)
    assert np.array_equal(_groups(idx, a, b, s, s, 1.0), np.zeros(n, np.int64))
    assert np.array_equal(_groups(idx, a, b, s, s * 0.5, 1.0), np.arange(n))
    assert np.array_equal(_groups(idx, a[:0], b[:0], s[:0], s[:0], 1.0), np.arange(n))


def _planted(seed=23, n_base=24):
    """Random pages, noisy copies of a few of them, and a copy with 10 % of rows dropped."""
    rng = np.random.default_rng(seed)
    base = [_unit(rng, int(n)) for n in rng.integers(40, 200, size=n_base)]
    pages, planted = list(base), []
    for src in (2, 5, 11):
        near = base[src] + np.float32(0.05) * _unit(rng, len(base[src]))
        pages.append(near / np.linalg.norm(near, axis=1, keepdims=True))
        planted.append((src, len(pages) - 1))
    keep = rng.permutation(len(base[7]))[: int(0.9 * len(base[7]))]
    pages.append(base[7][np.sort(keep)])
    planted.append((7, len(pages) - 1))
    return pages, planted


def run(coro):
    return asyncio.run(coro)


def _store(dtype, **kw):
    """The planted pages as chunks of documents d0 .. d3; pages 20 .. 23 belong to app "a1" (visible to it alone)."""
    pages, planted = _planted()
    store = B200MultiVectorStore(mode=dtype, coalesce_queries=False, **kw)
    for lo, hi, app in ((0, 20, None), (20, 24, "a1"), (24, len(pages), None)):
        run(store.store_embeddings([DocumentChunk(document_id=f"d{i % 4}", chunk_number=i, content=str(i), embedding=pages[i],
                                                  metadata={}) for i in range(lo, hi)], app_id=app))
    return store, pages, planted


def _oracle_candidates(qp, kind, scale, n_cand):
    """Each page's top n_cand other pages by sim(source -> page) (score DESC, page ASC), canonicalised."""
    n = len(qp)
    a, b = np.meshgrid(np.arange(n), np.arange(n), indexing="ij")
    sims = pair_sims(qp, a.ravel(), b.ravel(), kind, scale)[0].reshape(n, n)
    src, dst = [], []
    for s in range(n):
        best = sorted((p for p in range(n) if p != s), key=lambda p: (-float(sims[s, p]), p))[:n_cand]
        src += [s] * len(best)
        dst += best
    return canonical_pairs(src, dst)


N_CAND = 5


@pytest.mark.parametrize("kw", [{}, {"fde_candidates": 64}, {"sign_candidates": 64}],
                         ids=["exhaustive", "fde", "sign"])
@pytest.mark.parametrize("dtype", ["bf16", "int8"])
def test_store_end_to_end(dtype, kw):
    if kw.get("sign_candidates") is None and kw and dtype == "int8":
        pytest.skip("one dtype per first stage")
    store, pages, planted = _store(dtype, **kw)
    n = len(pages)
    n_pairs = run(store.index_duplicates(n_candidates=N_CAND))
    idx = store._index
    d = store._dup
    a, b = d["a"].cpu().numpy(), d["b"].cpu().numpy()
    assert np.array_equal(np.stack(canonical_pairs(a, b)), np.stack([a, b])) and n_pairs == len(a)
    found = set(zip(a.tolist(), b.tolist()))
    assert all(p in found for p in planted), (planted, sorted(found))
    kind = KIND[dtype]
    qp = [quantise_rows(p, kind) for p in pages]
    if not kw and dtype == "int8":  # exhaustive on exact scores: exactly the oracle's pair set
        wa, wb = _oracle_candidates(qp, kind, idx.score_scale, N_CAND)
        assert np.array_equal(a, wa) and np.array_equal(b, wb)
    sab, sba = d["sab"].cpu().numpy(), d["sba"].cpu().numpy()
    # the table's sims against the oracle; the groups from the oracle's sims where they are exact
    w_ab, w_ba = pair_sims(qp, a, b, kind, idx.score_scale)
    if kind == "int8":
        assert np.array_equal(sab, w_ab) and np.array_equal(sba, w_ba)
    else:
        assert np.all(np.abs(sab - w_ab) <= TOL[dtype] * np.maximum(np.abs(w_ab), 1.0))
        assert np.all(np.abs(sba - w_ba) <= TOL[dtype] * np.maximum(np.abs(w_ba), 1.0))
    planted_set = set(planted)
    t = float(min(min(sab[i], sba[i]) for i in range(len(a)) if (a[i], b[i]) in planted_set))
    groups = run(store.find_duplicate_chunks(t))
    labels = union_find_labels(n, edges(a, b, sab, sba, t))
    want = [sorted(np.flatnonzero(labels == g).tolist()) for g in sorted(set(labels.tolist()))]
    want = [g for g in want if len(g) > 1]
    assert [[c.chunk_number for c in g] for g in groups] == want
    q = pages[5][:20]
    for filt in ({}, {"doc_ids": ["d0", "d1", "d3"]}, {"app_id": "a1"}, {"app_id": "other"},
                 {"doc_ids": ["d0", "d2"], "app_id": "other"}):
        flat = run(store.query_similar(q, k=n, **filt))
        scores = np.full(n, -np.inf)
        for c in flat:
            scores[c.chunk_number] = c.score
        allowed = np.isfinite(scores)
        if filt.get("app_id") == "other":
            assert not allowed[20:24].any()
        lab = union_find_labels(n, edges(a, b, sab, sba, t, allowed), allowed)
        got = run(store.query_similar_distinct(q, 6, t, **filt))
        assert [c.chunk_number for c in got] == collapsed_topk(scores, lab, 6), filt
        for c in got:
            assert c.score == np.float32(scores[c.chunk_number])
            others = sorted(o for o in np.flatnonzero(lab == lab[c.chunk_number]).tolist() if o != c.chunk_number)
            assert sorted(x[1] for x in c.metadata["duplicates"]) == others
        vis = [[c.chunk_number for c in g] for g in run(store.find_duplicate_chunks(t, **filt))]
        assert all(allowed[p] for g in vis for p in g), filt


def test_cross_stream_order():
    idx = _index("bf16")
    a, b = _pairs()
    ad, bd = _dev(a), _dev(b)
    s1, s2 = torch.cuda.Stream(), torch.cuda.Stream()
    alone_ab, alone_ba = idx.pair_maxsim(ad, bd)
    alone_lab = idx.duplicate_groups(ad, bd, alone_ab, alone_ba, 0.5)
    alone_search = idx.search_pages([12], 5)
    torch.cuda.synchronize()
    for _ in range(2):
        with torch.cuda.stream(s1):
            sab, sba = idx.pair_maxsim(ad, bd)
            lab = idx.duplicate_groups(ad, bd, sab, sba, 0.5)
        with torch.cuda.stream(s2):
            other = idx.search_pages([12], 5)
        torch.cuda.synchronize()
        assert torch.equal(sab.view(torch.int32), alone_ab.view(torch.int32))
        assert torch.equal(sba.view(torch.int32), alone_ba.view(torch.int32))
        assert torch.equal(lab, alone_lab)
        for x, y in zip(other, alone_search):
            assert torch.equal(x, y)


def test_refusals():
    idx = _index("bf16")
    with pytest.raises(ValueError):
        idx.duplicate_groups(_dev([0]), _dev([1]), _dev([1.0], torch.float32), _dev([1.0], torch.float32), float("nan"))
    with pytest.raises(ValueError):
        idx.pair_maxsim(_dev([0, 1]), _dev([1]))
    host = MaxSimIndex(dtype="bf16", tier="host")
    host.add_pages(PAGES[:3])
    from morphik_core_b200._native import NativeError

    with pytest.raises(NativeError):
        host.pair_maxsim(_dev([1]), _dev([2]))
