"""Every corpus dtype on every scoring path against the oracle (run with -m gpu on an H100).

The corpora are the planted-maximum corpora of oracle/planted.py: every page holds, for each query direction, one designated
row that is that direction's maximum by >= 0.25, placed on page / chunk / tile boundaries (tests/test_planted_corpus.py
shows on the CPU that deleting such a row or moving a page boundary by one row or one chunk moves a score far beyond the
tolerance).  So a scorer that drops a row or gives a boundary row to the neighbouring page or slot fails here, whatever the
random draw.  One random ragged corpus with empty pages covers zero_pad_compat, where the clamp needs negative maxima.

Paths: the full scan (NM = 1 / 2 / 4 / 8 resident query tiles, phantom tiles, several passes; max_ctas default / 1 / 3;
unit_rows default / 64 / 400), top-k with and without allow-masks, the shared-list and per-query reranks (duplicate ids,
-1 and ids past the corpus as unused slots, empty pages, queries of 1 .. 300 tokens), zero_pad_compat, and the two-level
(sliced) top-k of a rerank with exact ties.  Exhaustive value tests: every product of two finite e4m3 codes, of two int8
values in -127..127, and of an int8 query value with every packed code -128..127.
"""
import ctypes
import functools

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

torch = pytest.importorskip("torch")
if not torch.cuda.is_available():  # pragma: no cover - the gpu marker normally deselects these on CPU boxes
    pytest.skip("CUDA device required", allow_module_level=True)

from morphik_core_b200 import _native as nat  # noqa: E402
from morphik_core_b200.index import MaxSimIndex  # noqa: E402
from oracle import maxsim_oracle as orc  # noqa: E402
from oracle import planted  # noqa: E402
from oracle.scoring import (assert_candidate_ranking, assert_ranking, assert_scores, oracle_scores,  # noqa: E402
                            slot_scores_of)

# (corpus dtype, b1_tensor option): 1-bit full scans run on the POPC kernel (0) or the wgmma kernel with bit expansion (1)
KINDS = {"bf16": ("bf16", None), "int8": ("int8", None), "fp8": ("fp8", None), "b1_popc": ("binary", 0),
         "b1_wgmma": ("binary", 1)}

# query batches by the query tiles (4 x 32-token groups) they fill
BATCHES = {
    "nm1": [32],                                   # 1 group: one busy warp
    "nm2": [32, 40, 1, 64],                        # 6 groups, 2 tiles
    "nm4_phantom": [130, 33, 5, 7, 20, 31],        # 11 groups, 3 tiles -> NM = 4 with a phantom tile
    "nm8": [32 if i % 3 else 17 for i in range(30)],  # 30 groups, 8 tiles: int8 / 1-bit NM = 8, bf16 / fp8 two passes
    "passes": [300] + [32 if i % 2 else 29 for i in range(60)],  # 70 groups, 18 tiles: several passes
}
# per-query rerank: four 1-group queries share tile 0, then 1 / 33 / 130 tokens, and 300 tokens spanning three tiles
RERANK_T = [5, 17, 32, 9, 1, 33, 130, 300]


@functools.lru_cache(maxsize=None)
def corpus(dtype):
    return planted.planted_corpus(dtype, seed=2024, n_random=40)


@functools.lru_cache(maxsize=None)
def queries(dtype, name):
    return planted.planted_queries(corpus(dtype), BATCHES[name] if name in BATCHES else RERANK_T, seed=len(name))


@functools.lru_cache(maxsize=None)
def oracle(dtype, name):
    return oracle_scores(dtype, queries(dtype, name), corpus(dtype).pages)


def make_index(kind, pages, unit_rows=0, zero_pad=0):
    dtype, b1 = KINDS[kind]
    idx = MaxSimIndex(dtype=dtype)
    if b1 is not None:
        idx.set_option("b1_tensor", b1)
    if unit_rows:
        idx.set_option("unit_rows", unit_rows)
    if zero_pad:
        idx.set_option("zero_pad_compat", zero_pad)
    idx.add_pages(pages)
    return idx


def rerank_shared(idx, qs, cand, k):
    """b200ms_rerank_device: one candidate list for every query."""
    idx._attach()
    qd = torch.from_numpy(np.concatenate(qs).astype(np.float32)).cuda()
    cd = torch.from_numpy(np.asarray(cand, dtype=np.int64)).cuda()
    n_q = len(qs)
    ts = torch.empty((n_q, k), dtype=torch.float32, device="cuda")
    ti = torch.empty((n_q, k), dtype=torch.int64, device="cuda")
    tc = torch.empty((n_q,), dtype=torch.int32, device="cuda")
    vp = lambda t: ctypes.c_void_p(t.data_ptr())  # noqa: E731
    idx.h.check(nat.lib.b200ms_rerank_device(idx.h.ptr, vp(qd), nat.F32, nat.i32_array([len(q) for q in qs]), n_q, vp(cd),
                                             len(cand), k, ctypes.c_float(idx.i8_scale), ctypes.c_float(idx.score_scale),
                                             vp(ts), vp(ti), vp(tc), idx._stream()), "b200ms_rerank_device")
    torch.cuda.synchronize()
    return ts.cpu().numpy(), ti.cpu().numpy(), tc.cpu().numpy()


def rerank_per_query(idx, qs, cand, k):
    qd = torch.from_numpy(np.concatenate(qs).astype(np.float32)).cuda()
    ts, ti, tc = idx.rerank_batch(qd, [len(q) for q in qs], torch.from_numpy(np.ascontiguousarray(cand, np.int64)).cuda(), k)
    torch.cuda.synchronize()
    return ts.cpu().numpy(), ti.cpu().numpy(), tc.cpu().numpy()


def candidate_lists(rng, n_pages, n_lists, n_cand, empty_pages):
    """Random candidate lists with duplicates, unused slots (-1), ids past the corpus and empty pages."""
    cand = np.stack([rng.permutation(n_pages)[:n_cand] for _ in range(n_lists)]).astype(np.int64)
    for i in range(n_lists):
        cand[i, 3] = cand[i, 1]                     # duplicate id (tie: the earlier slot first)
        cand[i, n_cand - 1] = cand[i, 0]
        cand[i, 5] = -1
        cand[i, 8] = n_pages                        # past the corpus: unused
        cand[i, 9 + i % 5] = n_pages + 1000 * i + 7
        cand[i, 20] = empty_pages[i % len(empty_pages)]
    return cand


# ------------------------------------------------------------------------------------------------ full scan
@pytest.mark.parametrize("unit_rows", [0, 64, 400])
@pytest.mark.parametrize("kind", list(KINDS))
def test_full_scan_matches_oracle(kind, unit_rows):
    dtype = KINDS[kind][0]
    idx = make_index(kind, corpus(dtype).pages, unit_rows)
    for name in BATCHES:
        want = oracle(dtype, name)
        for max_ctas in (0, 1, 3):
            idx.set_option("max_ctas", max_ctas)
            got = idx.score_matrix(queries(dtype, name))
            assert_scores(dtype, got, want, f"{kind} unit_rows={unit_rows} {name} max_ctas={max_ctas}")


def test_random_ragged_corpus_with_empty_pages():
    """The planted corpora's lengths are >= 8 rows; here pages of 1 .. 1030 rows and runs of empty pages, every kind."""
    rng = np.random.default_rng(17)
    lens = [1, 0, 0, 2, 31, 32, 33, 0, 7] + [int(x) for x in rng.integers(1, 300, size=60)] + [1030, 0, 1]
    pages = [(rng.standard_normal((n, 128)) / np.sqrt(128)).astype(np.float32) for n in lens]
    qs = [(rng.standard_normal((t, 128)) / np.sqrt(128)).astype(np.float32) for t in (32, 7, 130, 1, 64)]
    for kind, (dtype, _) in KINDS.items():
        want = oracle_scores(dtype, qs, pages)
        for unit_rows in (0, 64):
            got = make_index(kind, pages, unit_rows).score_matrix(qs)
            assert_scores(dtype, got, want, f"{kind} unit_rows={unit_rows}")
            assert np.all(got[:, [p for p, n in enumerate(lens) if n == 0]] == 0.0)


# ------------------------------------------------------------------------------------------------ top-k
@pytest.mark.parametrize("kind", list(KINDS))
def test_topk_matches_oracle_order(kind):
    dtype = KINDS[kind][0]
    pc = corpus(dtype)
    idx = make_index(kind, pc.pages)
    rng = np.random.default_rng(3)
    n_pages = len(pc.pages)
    allowed = rng.random(n_pages) < 0.5
    others = [rng.random(n_pages) < f for f in (0.2, 0.9)]
    for name in ("nm1", "nm4_phantom"):
        qs, want = queries(dtype, name), oracle(dtype, name)
        for k in (1, 10, n_pages + 5):
            ts, ti, tc = idx.search_host(qs, k=k)
            for qi in range(len(qs)):
                assert_ranking(dtype, ts[qi], ti[qi], tc[qi], want[qi], k, what=f"{kind} {name} k={k} q{qi}")
            ts, ti, tc = idx.search_host(qs, k=k, allow_mask=idx.mask_from_pages(allowed))
            for qi in range(len(qs)):
                assert_ranking(dtype, ts[qi], ti[qi], tc[qi], want[qi], k, allowed, f"{kind} {name} masked k={k} q{qi}")
        masks = [None if qi % 3 == 0 else (allowed, *others)[qi % 3] for qi in range(len(qs))]
        ts, ti, tc = idx.search_host_masked(qs, 10, [None if m is None else idx.mask_from_pages(m) for m in masks])
        for qi in range(len(qs)):
            assert_ranking(dtype, ts[qi], ti[qi], tc[qi], want[qi], 10, masks[qi], f"{kind} {name} per-query mask q{qi}")


# ------------------------------------------------------------------------------------------------ reranks
@pytest.mark.parametrize("dtype", ["bf16", "int8", "fp8", "binary"])
def test_reranks_match_oracle_on_candidates(dtype):
    pc = corpus(dtype)
    kind = "b1_popc" if dtype == "binary" else dtype
    idx = make_index(kind, pc.pages)
    n_pages = len(pc.pages)
    empty = [p for p, n in enumerate(pc.lens) if n == 0]
    qs, want = queries(dtype, "rerank"), oracle(dtype, "rerank")
    rng = np.random.default_rng(8)
    n_cand = 48
    per_q = candidate_lists(rng, n_pages, len(qs), n_cand, empty)
    shared = candidate_lists(rng, n_pages, 1, n_cand, empty)[0]
    for k in (7, n_cand):
        ts, ti, tc = rerank_per_query(idx, qs, per_q, k)
        for qi in range(len(qs)):
            assert_candidate_ranking(dtype, ts[qi], ti[qi], tc[qi], slot_scores_of(want[qi], per_q[qi]), per_q[qi], n_pages,
                                     k, f"per-query {dtype} k={k} q{qi} ({len(qs[qi])} tokens)")
        ts, ti, tc = rerank_shared(idx, qs, shared, k)
        for qi in range(len(qs)):
            assert_candidate_ranking(dtype, ts[qi], ti[qi], tc[qi], slot_scores_of(want[qi], shared), shared, n_pages, k,
                                     f"shared {dtype} k={k} q{qi} ({len(qs[qi])} tokens)")


# ------------------------------------------------------------------------------------------------ zero_pad_compat
@pytest.mark.parametrize("batch", [3, 128])
@pytest.mark.parametrize("dtype", ["bf16", "int8", "fp8"])
def test_zero_pad_compat_full_scan_and_reranks(dtype, batch):
    """Non-negative pages and partly all-negative queries: many true maxima are negative, so the clamp of short pages
    shows.  Full scans batch pages in page-id order; reranks batch the candidate slots of each list in list order."""
    rng = np.random.default_rng(29 + batch)
    lens = [int(x) for x in rng.integers(1, 200, size=150)] + [0, 400, 3]
    lens[7] = lens[40] = 0
    pages = [(np.abs(rng.standard_normal((n, 128))) / np.sqrt(128)).astype(np.float32) for n in lens]
    qs = [(rng.standard_normal((t, 128)) / np.sqrt(128) * (-1.0 if i % 2 else 1.0)).astype(np.float32) for i, t in
          enumerate((20, 32, 1, 45, 130))]
    qs[1] = -np.abs(qs[1])
    qs[3] = -np.abs(qs[3])
    idx = make_index(dtype, pages, zero_pad=batch)
    want = oracle_scores(dtype, qs, pages, batch)
    clean = oracle_scores(dtype, qs, pages)
    assert np.abs(want - clean).max() > 0.05  # the clamp changes scores
    for max_ctas in (0, 3):
        idx.set_option("max_ctas", max_ctas)
        assert_scores(dtype, idx.score_matrix(qs), want, f"zero_pad {dtype} batch={batch} max_ctas={max_ctas}")
    # reranks: the clamp follows each candidate list (unused slots count as empty pages of their batch)
    n_pages = len(pages)
    cand = candidate_lists(rng, n_pages, len(qs), 40, [7, 40, 150])
    ts, ti, tc = rerank_per_query(idx, qs, cand, 40)
    for qi, q in enumerate(qs):
        sub = [pages[c] if 0 <= c < n_pages else pages[7] for c in cand[qi]]
        slot_want = oracle_scores(dtype, [q], sub, batch)[0]
        assert_candidate_ranking(dtype, ts[qi], ti[qi], tc[qi], slot_want, cand[qi], n_pages, 40, f"per-query zp q{qi}")
    shared = cand[0]
    sub = [pages[c] if 0 <= c < n_pages else pages[7] for c in shared]
    slot_want = oracle_scores(dtype, qs, sub, batch)
    ts, ti, tc = rerank_shared(idx, qs, shared, 40)
    for qi in range(len(qs)):
        assert_candidate_ranking(dtype, ts[qi], ti[qi], tc[qi], slot_want[qi], shared, n_pages, 40, f"shared zp q{qi}")


# ------------------------------------------------------------------------------------------------ sliced candidate top-k
@pytest.mark.parametrize("k", [10, 1000])
def test_sliced_candidate_topk_breaks_ties_by_slot(k):
    """20000 candidates select through the two-level top-k (per-slice select + merge).  A 1-bit corpus of 40 distinct
    pages repeated, candidates drawn with repetition: thousands of exact ties, which must come out in slot order (the
    better first-stage rank first), not in page-id order."""
    rng = np.random.default_rng(4)
    distinct = [np.where(rng.random((4, 128)) < 0.5, -1.0, 1.0).astype(np.float32) for _ in range(40)]
    n_pages = 3000
    pages = [distinct[p % 40] for p in range(n_pages)]
    idx = make_index("b1_popc", pages)
    qs = [distinct[3][:2].copy(), np.where(rng.random((9, 128)) < 0.5, -1.0, 1.0).astype(np.float32)]
    want = oracle_scores("binary", qs, pages)
    n_cand = 20000
    cand = rng.integers(0, n_pages, size=(2, n_cand)).astype(np.int64)
    cand[:, 100:110] = -1
    cand[:, 200] = n_pages + 5
    ts, ti, tc = rerank_shared(idx, qs, cand[0], k)
    for qi in range(2):
        assert_candidate_ranking("binary", ts[qi], ti[qi], tc[qi], slot_scores_of(want[qi], cand[0]), cand[0], n_pages, k,
                                 f"shared q{qi}")
    ts, ti, tc = rerank_per_query(idx, qs, cand, k)
    for qi in range(2):
        assert_candidate_ranking("binary", ts[qi], ti[qi], tc[qi], slot_scores_of(want[qi], cand[qi]), cand[qi], n_pages, k,
                                 f"per-query q{qi}")


# ------------------------------------------------------------------------------------------------ exhaustive value sets
def test_fp8_every_product_of_two_finite_codes_is_exact():
    """Query a: one token whose only nonzero element (a mod 128) is deq(a)/64; page b: one row of deq(b)/64 everywhere.
    Every score is the single product deq(a) * deq(b) / 64^2, exact in fp32 (padding tokens add 0)."""
    codes = np.asarray([c for c in range(256) if c & 0x7F != 0x7F], dtype=np.uint8)  # 254 finite e4m3 codes
    vals = orc.dequantize_e4m3_np(codes).astype(np.float64)
    qs = []
    for c, v in zip(codes, vals):
        q = np.zeros((1, 128), np.float32)
        q[0, int(c) % 128] = v / 64.0
        qs.append(q)
    pages = [np.full((1, 128), v / 64.0, np.float32) for v in vals]
    idx = MaxSimIndex(dtype="fp8")
    idx.add_pages(pages)
    packed = idx.packed_rows().cpu().numpy()
    assert np.array_equal(packed[::32], np.repeat(codes[:, None], 128, axis=1))  # page b's row (and its padding) = code b
    scores, goff, n_pages, q_packed = idx.score_groups(qs)
    torch.cuda.synchronize()
    qp = q_packed.cpu().numpy().reshape(-1, 128)[: 32 * len(codes): 32]
    want_q = np.zeros((len(codes), 128), np.uint8)
    want_q[np.arange(len(codes)), codes.astype(np.int64) % 128] = codes
    nonzero = (codes & 0x7F) != 0
    assert np.array_equal(qp[nonzero], want_q[nonzero])  # query codes too (+-0 rows: any zero code)
    assert np.all(qp[~nonzero] & 0x7F == 0)
    got = idx.score_matrix(qs)
    want = np.outer(vals, vals) / 4096.0
    bad = np.argwhere(got != want)
    assert not len(bad), [(int(codes[a]), int(codes[b]), got[a, b], want[a, b]) for a, b in bad[:5]]


def test_int8_every_product_of_two_values_is_exact():
    """The same construction over int8 values -127 .. 127: score = a * b exactly.  The quantiser never writes -128, but
    packed rows may hold it: a second corpus of every code -128 .. 127, loaded through append_packed, must give every
    product of a query value and a code exactly too."""
    vals = np.arange(-127, 128)
    qs = []
    for a in vals:
        q = np.zeros((1, 128), np.float32)
        q[0, int(a) % 128] = a / 127.0
        qs.append(q)
    pages = [np.full((1, 128), b / 127.0, np.float32) for b in vals]
    idx = MaxSimIndex(dtype="int8")
    idx.add_pages(pages)
    packed = idx.packed_rows().cpu().numpy().view(np.int8)
    assert np.array_equal(packed[::32], np.repeat(vals[:, None], 128, axis=1).astype(np.int8))
    scores, goff, n_pages, _ = idx.score_groups(qs)
    torch.cuda.synchronize()
    raw = scores[: len(vals), :n_pages].cpu().numpy().astype(np.int64)
    assert np.array_equal(goff[:-1], np.arange(len(vals)))
    want = np.outer(vals, vals)
    bad = np.argwhere(raw != want)
    assert not len(bad), [(int(vals[a]), int(vals[b]), raw[a, b], want[a, b]) for a, b in bad[:5]]
    codes = np.arange(-128, 128)
    rows = np.repeat(np.repeat(codes[:, None], 128, axis=1), 32, axis=0).astype(np.int8)  # page c: 32 rows of code c
    every = MaxSimIndex(dtype="int8")
    every.append_packed(torch.from_numpy(rows.view(np.uint8)).cuda(), [1] * len(codes))
    assert np.array_equal(every.packed_rows().cpu().numpy().view(np.int8)[::32, 0], codes.astype(np.int8))
    scores, goff, n_pages, _ = every.score_groups(qs)
    torch.cuda.synchronize()
    raw = scores[: len(vals), :n_pages].cpu().numpy().astype(np.int64)
    want = np.outer(vals, codes)
    bad = np.argwhere(raw != want)
    assert not len(bad), [(int(vals[a]), int(codes[b]), raw[a, b], want[a, b]) for a, b in bad[:5]]
