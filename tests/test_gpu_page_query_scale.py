"""Stored pages as queries on corpora past 4 GiB (-m gpu, H100): search_pages, page_rows, rerank_pages_batch, the example
calls, MMR and union_candidates, every page compared with a float64 reference.

The corpora are tests/scale_reference.py's planted corpora (bf16 20 480 pages, int8 / fp8 40 960, 1-bit 327 680), one
resident at a time, skipped with the reason when the card lacks the memory.  The reference is
page_query_oracle.page_query_reference: the source pages' packed bytes sliced from the corpus with torch (not by the library's
pack kernel), through scale_reference.reference_from_bytes, over the source's length.  Full scans read more than 1 GiB of
rows past byte 2^32; candidate lists, example pages and MMR candidates are asserted to lie (mostly) past it.
  * search_pages: 8 sources (past 4 GiB, the last page, a page near the start; about 260 query groups, several split
    launches) at k 10 and 4096, and with per-source masks, one of them allowing only pages past 4 GiB;
  * page_rows bit for bit against scale_reference.decode times the scale;
  * rerank_pages_batch of 1000 candidates, mostly past 4 GiB, with duplicates and unused slots; the int8 host tier bit for bit;
  * examples: two requests of query and page examples with +- weights: on 4096 candidates the fused scores are bit for bit a
    numpy float32 fusion of the device's own per-example scores; the full scan ranks within tolerance of the fusion of the
    reference rows (exactly for int8 and 1-bit);
  * MMR over 128 candidates past 4 GiB: every sim against the reference (exact for int8 and 1-bit), the picks replayed;
  * union_candidates of 8 lists of 4096 ids per request at width 4096 against a first-occurrence union.
"""
import gc
import time

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

torch = pytest.importorskip("torch")
if not torch.cuda.is_available():  # pragma: no cover - the gpu marker normally deselects these on CPU boxes
    pytest.skip("CUDA device required", allow_module_level=True)

import page_query_oracle as pqo  # noqa: E402
import scale_reference as sr  # noqa: E402
from morphik_core_b200 import _native as nat  # noqa: E402
from morphik_core_b200.index import MaxSimIndex  # noqa: E402
from oracle import maxsim_oracle as orc  # noqa: E402
from oracle.scoring import (TOL, assert_candidate_ranking, assert_ranking, i32_reported, i32_sum,  # noqa: E402
                            slot_scores_of)
from test_gpu_mmr import check_picks, run_mmr  # noqa: E402

DEV = torch.device("cuda", 0)
SEED = 0
PAGES = {"bf16": 20480, "int8": 40960, "fp8": 40960, "binary": 327680}
DTYPES = list(PAGES)
WORK_BYTES = 10 << 30
FOUR_GIB = 1 << 32
EXACT = ("int8", "binary")


def host(ts):
    torch.cuda.synchronize()
    return tuple(t.cpu().numpy() for t in ts)


def bits(x):
    return np.ascontiguousarray(x, np.float32).view(np.uint32)


class Corpus:
    def __init__(self, dtype):
        t0 = time.time()
        self.dtype = dtype
        self.idx = sr.build(dtype, PAGES[dtype], SEED)
        self.lens = np.asarray(self.idx.page_lens, dtype=np.int64)
        self.starts = pqo.starts_of(self.lens)
        self.rows = self.idx.packed_rows()
        self.rb = self.idx.row_bytes
        live = self.lens > 0
        self.past = np.flatnonzero((self.starts[:-1] * self.rb >= FOUR_GIB) & live)
        edge = [int(p) for p in self.past if self.lens[p] % 32 in (1, 31)][:1]
        rng = np.random.default_rng(5)
        self.src = ([int(np.flatnonzero(live)[1]), int(np.flatnonzero(live)[-1])] + edge +
                    [int(p) for p in rng.choice(self.past, 8 - 2 - len(edge), replace=False)])
        self.ref = pqo.page_query_reference(dtype, self.rows, self.lens, self.src)
        print(f"\n[page-query scale] {dtype}: {self.idx.n_pages} pages, {self.idx.n_rows_padded * self.rb / 2**30:.2f} GiB, "
              f"built and referenced in {time.time() - t0:.1f} s")

    def beyond(self, pages):
        """Bytes of the pages' rows past 2^32."""
        p = np.asarray(pages, np.int64)
        p = p[(p >= 0) & (p < len(self.lens))]
        end = (self.starts[p] + self.lens[p]) * self.rb
        return int(np.clip(end - np.maximum(self.starts[p] * self.rb, FOUR_GIB), 0, None).sum())

    def share_past(self, pages):
        """Share of the named pages' row bytes that lie past 2^32 (-1 slots ignored)."""
        p = np.asarray(pages, np.int64).ravel()
        p = p[(p >= 0) & (p < len(self.lens))]
        return self.beyond(p) / max(int(self.lens[p].sum()) * self.rb, 1)

    def sums(self, ref_row, n):
        """Exact dtypes: the integer sums behind reference scores over a length n."""
        return np.rint(np.asarray(ref_row) * n * sr._score_divisor(self.dtype)).astype(np.int64)

    def reported(self, ref_row, n):
        """Exact dtypes: the bits the device reports for reference scores over a length n (fp32(S * scale) / n)."""
        return i32_reported(self.sums(ref_row, n), self.idx.score_scale) / np.float32(n)


@pytest.fixture(scope="module")
def scale(request):
    dtype = request.param
    rows = int(sr.padded_rows(sr.page_lens(PAGES[dtype], SEED)).sum())
    gc.collect()
    torch.cuda.empty_cache()
    free, _ = torch.cuda.mem_get_info(DEV)
    need = rows * sr.ROW_BYTES[dtype] + WORK_BYTES
    if free < need:
        pytest.skip(f"the {dtype} corpus needs {need / 2**30:.1f} GiB of device memory, {free / 2**30:.1f} GiB are free")
    torch.cuda.reset_peak_memory_stats(DEV)
    c = Corpus(dtype)
    assert c.idx.n_rows_padded * c.rb > FOUR_GIB + (1 << 30)
    yield c
    print(f"\n[page-query scale] {dtype}: torch.cuda.max_memory_allocated = "
          f"{torch.cuda.max_memory_allocated(DEV) / 2**30:.2f} GiB")
    c.idx.close()
    del c
    gc.collect()
    torch.cuda.empty_cache()


def check_top(c, i, ts, ti, tc, k, allow=None, what=""):
    """Float dtypes: oracle.scoring's ranking check.  Exact dtypes: the ids of the exact sums' order and the reported bits
    (a score over the length is not a multiple of the score quantum, so assert_ranking's quantum check does not apply)."""
    want, n_src = c.ref[i], c.lens[c.src[i]]
    if c.dtype not in EXACT:
        return assert_ranking(c.dtype, ts, ti, tc, want, k, allow, what)
    _, wi = orc.topk_np(i32_sum(c.sums(want, n_src)).astype(np.float64), k, allow)
    n = len(wi)
    assert int(tc) == n and np.array_equal(ti[:n], wi) and (ti[n:] == -1).all(), what
    assert np.array_equal(bits(ts[:n]), bits(c.reported(want, n_src)[wi])), what


@pytest.mark.parametrize("scale", DTYPES, indirect=True)
def test_search_pages_and_page_rows(scale):
    c = scale
    assert c.beyond(np.arange(c.idx.n_pages)) >= 1 << 30  # a full scan reads every page
    print(f"\n[page-query scale] {c.dtype}: {c.share_past(c.src):.0%} of the source rows past 4 GiB")
    groups = sum((int(c.lens[p]) + 31) // 32 for p in c.src)
    assert groups >= 200, groups
    for k in (10, 4096):
        ts, ti, tc = host(c.idx.search_pages(c.src, k))
        for i, p in enumerate(c.src):
            check_top(c, i, ts[i], ti[i], tc[i], k, what=f"{c.dtype} search_pages k={k} source {p}")
    n = c.idx.n_pages
    rng = np.random.default_rng(2)
    past = np.zeros(n, bool)
    past[c.past] = True
    rows = [rng.random(n) < 0.01, past]
    masks = torch.from_numpy(np.stack([c.idx.mask_from_pages(r) for r in rows]).view(np.int32)).to(DEV)
    index = [1, 0, -1, 1, 0, 1, 1, -1]
    ts, ti, tc = host(c.idx.search_pages(c.src, 4096, masks, torch.tensor(index, dtype=torch.int32, device=DEV)))
    for i, p in enumerate(c.src):
        allow = rows[index[i]] if index[i] >= 0 else None
        check_top(c, i, ts[i], ti[i], tc[i], 4096, allow, f"{c.dtype} masked source {p} row {index[i]}")
    # page_rows: the sources' rows decoded and scaled in float32
    got, lens = c.idx.page_rows(c.src)
    scale_f = 1.0 / c.idx.i8_scale if c.dtype in ("int8", "fp8") else 1.0
    want = torch.cat([sr.decode(c.dtype, c.rows[c.starts[p]:c.starts[p] + c.lens[p]], torch.float32) for p in c.src])
    want = want * torch.tensor(scale_f, dtype=torch.float32, device=DEV)
    assert torch.equal(got[:sum(lens)].view(torch.int32), want.view(torch.int32))


def candidate_lists(c, n_q, n_cand, seed):
    """Mostly pages past 4 GiB, some from anywhere, an empty page, the last page, duplicates and -1 slots."""
    rng = np.random.default_rng(seed)
    n = c.idx.n_pages
    cand = np.where(rng.random((n_q, n_cand)) < 0.9, rng.choice(c.past, (n_q, n_cand)), rng.integers(0, n, (n_q, n_cand)))
    cand[:, 3] = cand[:, 1]
    cand[:, n_cand - 1] = cand[:, 0]
    cand[:, 5] = -1
    cand[:, 600] = -1
    cand[:, 7] = np.flatnonzero(c.lens == 0)[-1]
    cand[:, 8] = n - 1
    return np.ascontiguousarray(cand, dtype=np.int64)


@pytest.mark.parametrize("scale", DTYPES, indirect=True)
def test_rerank_pages_batch(scale):
    c = scale
    n = c.idx.n_pages
    cand = candidate_lists(c, len(c.src), 1000, 11)
    share = c.share_past(cand)
    print(f"\n[page-query scale] {c.dtype}: {share:.0%} of the candidate rows past 4 GiB")
    assert share >= 0.8
    cd = torch.from_numpy(cand).to(DEV)
    for k in (10, 1000):
        ts, ti, tc = host(c.idx.rerank_pages_batch(c.src, cd, k))
        for i, p in enumerate(c.src):
            what = f"{c.dtype} rerank_pages_batch k={k} source {p}"
            if c.dtype not in EXACT:
                assert_candidate_ranking(c.dtype, ts[i], ti[i], tc[i], slot_scores_of(c.ref[i], cand[i]), cand[i], n, k,
                                         what)
                continue
            valid = (cand[i] >= 0) & (cand[i] < n)
            keys = i32_sum(c.sums(slot_scores_of(c.ref[i], cand[i]), c.lens[p])).astype(np.float64)
            _, slots = orc.topk_np(keys, k, valid)
            m = len(slots)
            assert int(tc[i]) == m and np.array_equal(ti[i, :m], cand[i][slots]), what
            assert np.array_equal(bits(ts[i, :m]), bits(c.reported(c.ref[i], c.lens[p])[cand[i][slots]])), what
    if c.dtype != "int8":
        return
    hst = MaxSimIndex(dtype="int8", tier="host")
    try:
        hst.reserve_rows(c.idx.n_rows_padded)
    except nat.NativeError as e:
        hst.close()
        pytest.skip(f"no pinned host block of {c.idx.n_rows_padded * c.rb / 2**30:.1f} GiB: {e}")
    try:
        hst.append_packed(c.rows, c.idx._page_lens)
        for k in (10, 1000):
            want = host(c.idx.rerank_pages_batch(c.src, cd, k))
            got = host(hst.rerank_pages_batch(c.src, cd, k))
            for x, y in zip(got, want):
                assert np.array_equal(x.view(np.uint8), y.view(np.uint8)), f"host tier k={k}"
    finally:
        hst.close()


# ------------------------------------------------------------------------------------------------ examples
Q_TOKENS = [40, 33]


def example_call(c):
    """Two requests: query examples first (one per request), then page examples past 4 GiB; +- weights."""
    qs = sr.queries(c.dtype, SEED, Q_TOKENS, q_seed=3)
    pages = [int(c.past[-1]), int(c.past[len(c.past) // 2]), int(c.past[7])]
    ex_req = [0, 1, 0, 0, 1]
    w = [1.0, -0.25, -0.5, 0.75, 1.0]
    return qs, pages, ex_req, w


def query_reference(c, qs):
    """float64 [n_q, n_pages]: the reference of query examples over their token count."""
    _, goff, _, q_packed = c.idx.score_groups(qs)
    ref = sr.reference_scores(c.idx, q_packed, goff, [len(q) for q in qs])
    return ref / np.asarray([len(q) for q in qs], np.float64)[:, None]


@pytest.mark.parametrize("scale", DTYPES, indirect=True)
def test_examples(scale):
    c = scale
    n = c.idx.n_pages
    qs, pages, ex_req, w = example_call(c)
    assert c.share_past(pages) == 1.0 and c.beyond(np.arange(n)) >= 1 << 30
    q_dev = torch.from_numpy(np.concatenate(qs).astype(np.float32)).to(DEV)
    # candidate mode: every example's own rows, fused in numpy, are the device's fused rows bit for bit
    cand = candidate_lists(c, 2, 4096, 21)
    cd = torch.from_numpy(cand).to(DEV)
    ts, ti, tc = host(c.idx.rerank_batch(q_dev, Q_TOKENS, cd, 4096))
    per = {}
    for e in range(2):
        per[e] = dict(zip(ti[e, :tc[e]].tolist(), (ts[e, :tc[e]] / np.float32(Q_TOKENS[e])).tolist()))
    for j, p in enumerate(pages):
        r = ex_req[2 + j]
        s, i_, t = host(c.idx.rerank_pages_batch([p], cd[r:r + 1].contiguous(), 4096))
        per[2 + j] = dict(zip(i_[0, :t[0]].tolist(), s[0, :t[0]].tolist()))
    gs, gi, gc_ = host(c.idx.rerank_examples_batch(q_dev, Q_TOKENS, pages, ex_req, w, 2, cd, 4096))
    for r in range(2):
        mine = [e for e in range(5) if ex_req[e] == r]
        ids = gi[r, :gc_[r]]
        rows = np.stack([np.asarray([per[e][int(p)] for p in ids], np.float32) for e in mine])
        fused = pqo.fuse(rows, [w[e] for e in mine])
        assert np.array_equal(bits(gs[r, :gc_[r]]), bits(fused)), (c.dtype, r)
        assert int(gc_[r]) == int((cand[r] >= 0).sum())
    # full scan against the fusion of the reference rows
    ref = np.concatenate([query_reference(c, qs), pqo.page_query_reference(c.dtype, c.rows, c.lens, pages)])
    ts, ti, tc = host(c.idx.search_examples(q_dev, Q_TOKENS, pages, ex_req, w, 2, 4096))
    lens = Q_TOKENS + [int(c.lens[p]) for p in pages]
    for r in range(2):
        mine = [e for e in range(5) if ex_req[e] == r]
        what = f"{c.dtype} search_examples request {r}"
        assert int(tc[r]) == 4096, what
        if c.dtype in EXACT:
            fused = pqo.fuse(np.stack([c.reported(ref[e], lens[e]) for e in mine]), [w[e] for e in mine])
            _, wi = orc.topk_np(fused.astype(np.float64), 4096)
            assert np.array_equal(ti[r], wi) and np.array_equal(bits(ts[r]), bits(fused[wi])), what
            continue
        fused = sum(w[e] * ref[e] for e in mine)
        slack = 4 * TOL[c.dtype] * sum(abs(w[e]) * np.abs(ref[e]) for e in mine) + 1e-6
        assert (np.abs(ts[r] - fused[ti[r]]) <= slack[ti[r]]).all(), what
        rest = np.ones(n, bool)
        rest[ti[r]] = False
        assert (fused[rest] <= ts[r, -1] + slack[rest]).all(), what  # nothing left out beats the last pick


# ------------------------------------------------------------------------------------------------ MMR and union
@pytest.mark.parametrize("scale", DTYPES, indirect=True)
def test_mmr_past_4gib(scale):
    c = scale
    rng = np.random.default_rng(8)
    ids = np.sort(rng.choice(c.past, 128, replace=False)).astype(np.int64)[None]
    assert c.share_past(ids) == 1.0
    scores = rng.random((1, 128)).astype(np.float32) * 40
    k, lam = 12, 0.6
    got = run_mmr(c.idx, ids, scores, [40], k, lam)
    check_picks(ids, scores, [40], k, lam, got, c.idx.n_pages)
    # the candidates as a corpus of their own: sim(j -> s) = the reference of j's rows against page s
    sub_lens = c.lens[ids[0]]
    sub = torch.cat([c.rows[c.starts[p]:c.starts[p] + (sub_lens[j] + 31) // 32 * 32] for j, p in enumerate(ids[0])])
    ref = pqo.page_query_reference(c.dtype, sub, sub_lens, list(range(128)))
    gi, _, gcount, sims = got
    slot = {int(p): j for j, p in enumerate(ids[0])}
    live = np.ones(128, bool)
    for i in range(int(gcount[0])):
        s = slot[int(gi[0, i])]
        live[s] = False
        g = sims[0, i]
        assert np.isneginf(g[~live]).all()
        if c.dtype in EXACT:
            want = np.array([c.reported(ref[j, s:s + 1], sub_lens[j])[0] for j in range(128)], np.float32)
            assert np.array_equal(bits(g[live]), bits(want[live])), (c.dtype, i)
        else:
            want = ref[:, s]
            assert (np.abs(g[live] - want[live]) <= TOL[c.dtype] * np.maximum(np.abs(want[live]), 1e-3)).all(), (c.dtype, i)


@pytest.mark.parametrize("scale", ["int8"], indirect=True)
def test_union_candidates_past_4gib(scale):
    c = scale
    rng = np.random.default_rng(4)
    pool = rng.choice(c.past, 6000, replace=False)
    lists = rng.choice(pool, (16, 4096)).astype(np.int64)
    lists[:, ::97] = -1
    assert c.share_past(lists) == 1.0
    out = c.idx.union_candidates(torch.from_numpy(lists).to(DEV), [0, 8, 16], 4096).cpu().numpy()
    for r in range(2):
        seen, want = set(), []
        for p in lists[8 * r:8 * r + 8].ravel().tolist():
            if p >= 0 and p not in seen:
                seen.add(p)
                want.append(p)
        want = (want + [-1] * 4096)[:4096]
        assert out[r].tolist() == want, r
