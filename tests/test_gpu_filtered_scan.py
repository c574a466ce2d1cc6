"""A search with an allow mask scans only the pages the mask allows (run with -m gpu on an H100).

The filtered search builds its work units from the masks on the GPU (csrc/scan_plan.cu).  Three things are held here:
  * its results are bit for bit those of the path that scans everything: b200ms_score over the whole corpus, then
    b200ms_topk / b200ms_topk_docs with the same mask -- scores as bit patterns, ids and counts -- for every corpus dtype,
    every mask shape and every entry point that takes a mask, also right after a search that left other pages' scores in
    the handle's score matrix;
  * the plan it walked is the one tests/scan_plan_model.py derives (b200ms_last_scan_stats): the rows scanned are exactly
    the padded rows of the allowed pages;
  * one case per dtype is anchored to oracle.scoring.
The corpus is a planted corpus of oracle/planted.py (several thousand ragged pages, so that its scan is more than one wave of
work units and the filtered plan is taken) followed by pages of 0, 1, 2, 31 .. 1030 random rows.
"""
import ctypes
import functools

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

torch = pytest.importorskip("torch")
if not torch.cuda.is_available():  # pragma: no cover - the gpu marker normally deselects these on CPU boxes
    pytest.skip("CUDA device required", allow_module_level=True)

import scan_plan_model as spm  # noqa: E402
from morphik_core_b200 import _native as nat  # noqa: E402
from morphik_core_b200.index import MaxSimIndex  # noqa: E402
from oracle import planted  # noqa: E402
from oracle.scoring import assert_ranking, oracle_scores  # noqa: E402

DEV = torch.device("cuda", 0)
SMS = torch.cuda.get_device_properties(0).multi_processor_count
DTYPES = ["bf16", "int8", "fp8", "binary"]
# 1-bit full scans: one or two 32-token groups run on the POPC kernel (it walks the allowed-page list), three or more on wgmma
BATCHES = {"g1": [20], "g2": [33], "g11": [32, 40, 1, 64, 130]}
TAIL_LENS = [0, 1, 0, 0, 2, 31, 32, 33, 1030, 0, 1024, 1, 0]
K, PER_DOC, PAGES_PER_DOC = 12, 3, 16


def vp(t):
    return None if t is None else ctypes.c_void_p(t.data_ptr())


@functools.lru_cache(maxsize=None)
def corpus(dtype):
    pc = planted.planted_corpus(dtype, seed=77, n_random=2500)
    rng = np.random.default_rng(5)
    tail = [(rng.standard_normal((n, 128)) / np.sqrt(128)).astype(np.float32) for n in TAIL_LENS]
    return pc, pc.pages + tail


@functools.lru_cache(maxsize=None)
def queries(dtype, name):
    return planted.planted_queries(corpus(dtype)[0], BATCHES[name], seed=len(name))


@functools.lru_cache(maxsize=None)
def index(dtype, zero_pad=0):
    idx = MaxSimIndex(dtype=dtype)
    if zero_pad:
        idx.set_option("zero_pad_compat", zero_pad)
    idx.add_pages(corpus(dtype)[1])
    idx._attach()
    return idx


def lens_of(dtype):
    return [len(p) for p in corpus(dtype)[1]]


def mask_shapes(lens):
    """name -> bool [n_pages]"""
    n = len(lens)
    rng = np.random.default_rng(11)
    live = np.asarray(lens) > 0
    shapes = {}

    def only(pages):
        a = np.zeros(n, bool)
        a[pages] = True
        return a

    shapes["single"] = only([int(np.flatnonzero(live)[len(lens) // 3])])
    shapes["first"] = only([0])
    shapes["last"] = only([n - 1])
    shapes["document"] = only(list(range(1600, 1600 + PAGES_PER_DOC)))
    shapes["every_second"] = np.arange(n) % 2 == 0
    for pct in (1, 10, 50, 99):
        shapes[f"random_{pct}"] = rng.random(n) < pct / 100.0
    shapes["ones"] = np.ones(n, bool)
    shapes["zeros"] = np.zeros(n, bool)
    shapes["only_empty"] = ~live
    return shapes


def dev_words(words):
    return torch.from_numpy(np.ascontiguousarray(words).view(np.int32)).to(DEV)


def to_np(out):
    torch.cuda.synchronize()
    return [t.cpu().numpy() for t in out]


def assert_bits(got, want, what):
    assert len(got) == len(want)
    for i, (g, w) in enumerate(zip(got, want)):
        assert g.shape == w.shape and g.dtype == w.dtype, (what, i)
        assert np.array_equal(g.view(np.uint8), w.view(np.uint8)), f"{what}: output {i} differs from the scan of every page"


def q_dev(qs):
    return torch.from_numpy(np.concatenate(qs).astype(np.float32)).to(DEV)


def reference(idx, qs, allow_per_query, id_base=0, docs=None):
    """b200ms_score over every page, then b200ms_topk (docs = (page_doc, n_docs): b200ms_topk_docs) once per distinct mask;
    query i takes its rows from the call with allow_per_query[i] (bool [n_pages])."""
    n_q = len(qs)
    scores, goff, n_pages, _ = idx.score_groups(qs)
    assert idx.scan_stats() == {"units": len(spm.corpus_units(idx._page_lens, SMS, 4096)), "rows": idx._rows}
    goff_c = nat.i32_array(goff.tolist())
    sdt = nat.F32 if idx.float_scores else nat.I32
    ld, h, scale = scores.shape[1], idx.h, ctypes.c_float(idx.score_scale)
    shape = (n_q, K, PER_DOC) if docs else (n_q, K)
    final = None
    for key in sorted({a.tobytes() for a in allow_per_query}):
        rows = [i for i, a in enumerate(allow_per_query) if a.tobytes() == key]
        mask = dev_words(idx.mask_from_pages(allow_per_query[rows[0]]))
        out = [torch.empty(shape, dtype=torch.float32, device=DEV), torch.empty(shape, dtype=torch.int64, device=DEV)]
        if docs:
            out += [torch.empty((n_q, K), dtype=torch.int32, device=DEV), torch.empty((n_q,), dtype=torch.int32, device=DEV)]
            h.check(nat.lib.b200ms_topk_docs(h.ptr, vp(scores), sdt, n_pages, ld, goff_c, n_q, vp(mask), vp(docs[0]), docs[1], K,
                                             PER_DOC, scale, id_base, vp(out[0]), vp(out[1]), vp(out[2]), vp(out[3]),
                                             idx._stream()), "b200ms_topk_docs")
        else:
            out += [torch.empty((n_q,), dtype=torch.int32, device=DEV)]
            h.check(nat.lib.b200ms_topk(h.ptr, vp(scores), sdt, n_pages, ld, goff_c, n_q, vp(mask), K, scale, id_base, vp(out[0]),
                                        vp(out[1]), vp(out[2]), idx._stream()), "b200ms_topk")
        out = to_np(out)
        final = final or [np.empty_like(o) for o in out]
        for f, o in zip(final, out):
            f[rows] = o[rows]
    return final


def assert_plan(idx, masks, mask_index, what):
    """The plan the last search walked is the model's: its unit count, and exactly the allowed pages' padded rows."""
    p = spm.plan(masks, mask_index, idx._page_lens, SMS, 4096)
    allow = spm.allowed_pages(masks, mask_index, idx.n_pages)
    assert p.rows == int(spm.padded(idx._page_lens)[allow].sum())
    assert idx.scan_stats() == {"units": len(p.units), "rows": p.rows}, what


# ------------------------------------------------------------------------------------------------ one mask for every query
@pytest.mark.parametrize("dtype", DTYPES)
def test_masked_search_is_bit_identical_to_the_scan_of_every_page(dtype):
    idx = index(dtype)
    lens = lens_of(dtype)
    assert len(spm.corpus_units(lens, SMS, 4096)) > SMS  # more than one wave of units: the filtered plan is taken
    for shape, allow in mask_shapes(lens).items():
        words = idx.mask_from_pages(allow)
        for name in BATCHES:
            qs = queries(dtype, name)
            got = to_np(idx.search_device(q_dev(qs), BATCHES[name], K, allow_mask_dev=dev_words(words)))
            assert_plan(idx, words, None, f"{dtype} {shape} {name}")
            assert_bits(got, reference(idx, qs, [allow] * len(qs)), f"{dtype} {shape} {name}")
            if shape in ("zeros", "only_empty"):
                n = 0 if shape == "zeros" else min(K, int(allow.sum()))
                assert (got[2] == n).all() and (got[1][:, n:] == -1).all() and np.isneginf(got[0][:, n:]).all()
                assert (got[0][:, :n] == 0).all()  # pages without rows score 0


@pytest.mark.parametrize("dtype", DTYPES)
def test_bits_past_the_last_page_and_id_base(dtype):
    idx = index(dtype)
    assert idx.n_pages % 32  # the last mask word has spare bits
    allow = mask_shapes(lens_of(dtype))["random_10"]
    words = spm.mask_words(allow, set_tail=True)
    qs = queries(dtype, "g11")
    got = to_np(idx.search_device(q_dev(qs), BATCHES["g11"], K, allow_mask_dev=dev_words(words), id_base=1 << 40))
    assert_plan(idx, words, None, dtype)
    assert_bits(got, reference(idx, qs, [allow] * len(qs), id_base=1 << 40), dtype)


# ------------------------------------------------------------------------------------------------ per-query masks
@pytest.mark.parametrize("dtype", DTYPES)
def test_per_query_masks_scan_their_union(dtype):
    idx = index(dtype)
    shapes = mask_shapes(lens_of(dtype))
    rows = [shapes[s] for s in ("random_1", "document", "random_10", "only_empty")]
    masks = np.stack([idx.mask_from_pages(r) for r in rows])
    qs = queries(dtype, "g11")
    n_q = len(qs)
    for mask_index in ([0, 1, 2, 1, 3], [1, 1, 1, 1, 1], [3, 0, 0, 3, 0], [0, -1, 2, 1, 1]):
        mi = torch.tensor(mask_index, dtype=torch.int32, device=DEV)
        got = to_np(idx.search_device(q_dev(qs), BATCHES["g11"], K, allow_mask_dev=dev_words(masks), mask_index_dev=mi))
        assert_plan(idx, masks, mask_index, f"{dtype} {mask_index}")  # a query without a mask: the plan of every page
        allow = [rows[i] if i >= 0 else np.ones(idx.n_pages, bool) for i in mask_index]
        assert_bits(got, reference(idx, qs, allow), f"{dtype} {mask_index}")
    # the host entry points upload the same masks
    host = idx.search_host_masked(qs, K, [masks[i] for i in (0, 1, 2, 1, 3)])
    assert_plan(idx, masks, [0, 1, 2, 1, 3], f"{dtype} host")
    assert_bits(list(host), reference(idx, qs, [rows[i] for i in (0, 1, 2, 1, 3)]), f"{dtype} search_host_masked")
    host = idx.search_host(qs, K, allow_mask=masks[2])
    assert_bits(list(host), reference(idx, qs, [rows[2]] * n_q), f"{dtype} search_host")


@pytest.mark.parametrize("dtype", DTYPES)
def test_documents_of_a_filtered_scan(dtype):
    idx = index(dtype)
    n = idx.n_pages
    page_doc = (torch.arange(n, device=DEV, dtype=torch.int32) // PAGES_PER_DOC).contiguous()
    n_docs = (n + PAGES_PER_DOC - 1) // PAGES_PER_DOC
    shapes = mask_shapes(lens_of(dtype))
    qs = queries(dtype, "g11")
    for shape in ("document", "random_1", "random_50", "zeros"):
        words = idx.mask_from_pages(shapes[shape])
        got = to_np(idx.search_docs_device(q_dev(qs), BATCHES["g11"], K, PER_DOC, page_doc, n_docs, allow_mask_dev=dev_words(words)))
        assert_plan(idx, words, None, f"{dtype} docs {shape}")
        assert_bits(got, reference(idx, qs, [shapes[shape]] * len(qs), docs=(page_doc, n_docs)), f"{dtype} docs {shape}")


@pytest.mark.parametrize("dtype", ["bf16", "int8"])
def test_zero_pad_compat_clamp_follows_the_page_ids(dtype):
    idx = index(dtype, 128)
    shapes = mask_shapes(lens_of(dtype))
    qs = [-np.abs(q) if i % 2 else q for i, q in enumerate(queries(dtype, "g11"))]  # negative maxima: the clamp shows
    for shape in ("random_10", "every_second", "single"):
        words = idx.mask_from_pages(shapes[shape])
        got = to_np(idx.search_device(q_dev(qs), BATCHES["g11"], K, allow_mask_dev=dev_words(words)))
        assert_bits(got, reference(idx, qs, [shapes[shape]] * len(qs)), f"{dtype} zero_pad {shape}")


def test_sharded_search_of_one_rank():
    idx = index("bf16")
    idx.comm_init(bytes(128), 0, 1)
    shapes = mask_shapes(lens_of("bf16"))
    rows = [shapes["random_1"], shapes["document"]]
    masks = np.stack([idx.mask_from_pages(r) for r in rows])
    qs = queries("bf16", "g11")
    mask_index = [0, 1, 0, 0, 1]
    out = (torch.empty((5, K), dtype=torch.float32, device=DEV), torch.empty((5, K), dtype=torch.int64, device=DEV),
           torch.empty((5,), dtype=torch.int32, device=DEV))
    ticket = idx.sharded_search_begin(q_dev(qs), BATCHES["g11"], K, 0, out, allow_masks_dev=dev_words(masks),
                                      mask_index_dev=torch.tensor(mask_index, dtype=torch.int32, device=DEV))
    idx.sharded_search_end(ticket)
    got = to_np(out)
    assert_plan(idx, masks, mask_index, "sharded")
    assert_bits(got, reference(idx, qs, [rows[i] for i in mask_index]), "sharded_search_begin")


# ------------------------------------------------------------------------------------------------ stale scores
@pytest.mark.parametrize("dtype", DTYPES)
def test_scores_left_by_earlier_searches_are_never_returned(dtype):
    """The handle's score matrix keeps what earlier searches wrote for the pages a filtered scan skips."""
    idx = index(dtype)
    lens = np.asarray(lens_of(dtype))
    qs = queries(dtype, "g11")
    qd = q_dev(qs)
    top = to_np(idx.search_device(qd, BATCHES["g11"], K))[1]  # every page scored; these are the best ones
    best = np.unique(top[top >= 0])
    rng = np.random.default_rng(3)
    a = np.zeros(len(lens), bool)
    a[rng.choice(np.setdiff1d(np.flatnonzero(lens > 0), best), size=40, replace=False)] = True
    b = np.zeros(len(lens), bool)
    b[rng.choice(np.setdiff1d(np.flatnonzero(lens > 0), np.concatenate([best, np.flatnonzero(a)])), size=40, replace=False)] = True
    for name, allow in (("a", a), ("b", b), ("a again", a)):
        got = to_np(idx.search_device(qd, BATCHES["g11"], K, allow_mask_dev=dev_words(idx.mask_from_pages(allow))))
        assert allow[got[1][got[1] >= 0]].all()
        assert_bits(got, reference(idx, qs, [allow] * len(qs)), f"{dtype} after other searches: {name}")


# ------------------------------------------------------------------------------------------------ oracle
@pytest.mark.parametrize("dtype", DTYPES)
def test_filtered_search_matches_the_oracle(dtype):
    idx = index(dtype)
    pages = corpus(dtype)[1]
    allow = mask_shapes(lens_of(dtype))["random_10"]
    sub = np.flatnonzero(allow)
    for name in ("g1", "g11"):
        qs = queries(dtype, name)
        want = np.zeros((len(qs), len(pages)))
        want[:, sub] = oracle_scores(dtype, qs, [pages[p] for p in sub])
        ts, ti, tc = idx.search_host(qs, K, allow_mask=idx.mask_from_pages(allow))
        for qi in range(len(qs)):
            assert_ranking(dtype, ts[qi], ti[qi], tc[qi], want[qi], K, allow, f"{dtype} {name} q{qi}")


def test_a_mask_with_the_wrong_word_count_is_refused():
    idx = index("bf16")
    launches = int(nat.lib.b200ms_launch_count(idx.h.ptr))
    qs = queries("bf16", "g1")
    with pytest.raises(ValueError, match="words"):
        idx.search_device(q_dev(qs), BATCHES["g1"], K, allow_mask_dev=torch.zeros(idx.n_pages // 32, dtype=torch.int32, device=DEV))
    assert int(nat.lib.b200ms_launch_count(idx.h.ptr)) == launches


# ------------------------------------------------------------------------------------------------ stream order
# Modelled on tests/stream_order_cases.py: call A left in flight on one stream, call B issued on a second stream as soon as
# A returns, both on the same handle and so on the same plan scratch; both must return what they return alone.
def stream_cases():
    import test_gpu_stream_order as tso

    k = tso.K

    def filtered(row):
        def call(x, w):
            return tso.three(tso.TOPK, x.idx.search_device(x.q[w], tso.LENS[w], k, allow_mask_dev=x.masks[row].contiguous())), None
        return call

    def masked(x, w):  # every query filtered: the union of both rows is scanned
        mi = torch.tensor([i % 2 for i in range(len(tso.LENS[w]))], dtype=torch.int32, device=DEV)
        return tso.three(tso.TOPK, x.idx.search_device(x.q[w], tso.LENS[w], k, allow_mask_dev=x.masks, mask_index_dev=mi)), None

    def docs(x, w):
        return tso.three(tso.DOCS, x.idx.search_docs_device(x.q[w], tso.LENS[w], k, tso.PER_DOC, x.page_doc, x.n_docs,
                                                           allow_mask_dev=x.masks[1].contiguous())), None

    def host(x, w):
        return tso.three(tso.TOPK, x.idx.search_host(x.q_host[w], k, allow_mask=x.host_masks[w][1])), None

    return {"filtered-then-filtered": (filtered(0), filtered(1)), "unfiltered-then-filtered": (tso.c_search_device, filtered(1)),
            "filtered-then-unfiltered": (filtered(1), tso.c_search_device), "masked-then-docs": (masked, docs),
            "filtered-then-search_host": (filtered(0), host)}


STREAM_CASES = ["filtered-then-filtered", "unfiltered-then-filtered", "filtered-then-unfiltered", "masked-then-docs",
                "filtered-then-search_host"]


@pytest.mark.parametrize("kind", ["bf16", "int8", "b1_popc", "b1_wgmma"])
@pytest.mark.parametrize("case", STREAM_CASES)
def test_filtered_searches_in_flight_together_return_their_alone_results(case, kind):
    import test_gpu_stream_order as tso

    a, b = stream_cases()[case]
    x = tso.context(kind)
    s1, s2 = torch.cuda.Stream(DEV), torch.cuda.Stream(DEV)

    def run(fn, w, s):
        with torch.cuda.stream(s):
            return fn(x, w)[0]

    def alone(fn, w, s):
        x.reset()
        out = run(fn, w, s)
        torch.cuda.synchronize()
        return tso.to_host(out)

    want_a, want_b = alone(a, "a", s1), alone(b, "b", s2)
    x.reset()
    out_a = run(a, "a", s1)
    out_b = run(b, "b", s2)  # no synchronisation in between
    torch.cuda.synchronize()
    got_a, got_b = tso.to_host(out_a), tso.to_host(out_b)
    x.reset()
    tso.assert_same(got_a, want_a, f"A of {case} on S1")
    tso.assert_same(got_b, want_b, f"B of {case} issued while A ran")
