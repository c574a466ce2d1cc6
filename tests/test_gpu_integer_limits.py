"""The int8 and 1-bit scorers at their integer limits, on every path (run with -m gpu on an H100).

An int8 token scores at most 128 * 127^2 = 2 064 512, so a query of 1041 tokens of +-127 can pass 2^31 - 1 (1033 tokens
against rows of -128).  The I32 sum rule of include/b200ms.h: a page's sum is formed in int64 and clamped to +-(2^31 - 1);
pages inside the range rank exactly, pages beyond it tie at the bound (lower id or slot first), and the reported score is
float32(clamped sum) * scale.  Expected values come from the int64 oracles (oracle_int8_maxsim, oracle_binary_maxsim) with
oracle.scoring.i32_sum applied, and are compared with no tolerance: ids, counts, score bits and tie order.

  * Corpora from packed bytes (append_packed): pages of +127, -127, +64 (half magnitude), alternating-sign rows, empty
    pages, and a pair whose sums differ by exactly 1 above 2^24 (float32 reports them equal), the higher at the higher id.
  * Queries of +-1.0 rows (quantised to +-127) of 1, 33, 1040, 1041, 1042, 2080, 2081 and 4300 tokens, batched so that
    long and short queries share a call.
  * b200ms_topk and b200ms_topk_docs on group scores summing to 2^31 - 2, 2^31 - 1, one past it and far past both bounds,
    with the page at 2^31 - 1 above the page at 2^31 - 2 (float32 reports both as 2^31: only the order tells them apart).
  * Paths: b200ms_score + b200ms_topk (unit_rows default / 64, max_ctas 0 / 1 / 3), the filtered scan, search_host with a
    graph replay, search_device(_masked), both reranks (n_cand 4096 takes the sliced top-k), a full scan of 20 000 one-row
    pages (the sliced full-scan top-k), search_docs / rerank_docs, the host tier (bit-identical to HBM), the sign first
    stage into an int8 rerank, explain (raw integer token values sum in int64 to the oracle), and the store.
  * 1-bit corpora (POPC and wgmma full scans) at the same lengths, exact against the oracle; every int8 code, -128 included.
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

from docs_oracle import topk_docs_np  # noqa: E402
from morphik_core_b200 import _native as nat  # noqa: E402
from morphik_core_b200.index import MaxSimIndex  # noqa: E402
from morphik_core_b200.models import DocumentChunk  # noqa: E402
from morphik_core_b200.signs import SignTwoStageIndex  # noqa: E402
from morphik_core_b200.store import B200MultiVectorStore  # noqa: E402
from oracle import maxsim_oracle as orc  # noqa: E402
from oracle.scoring import I32_SUM_BOUND, i32_reported, i32_sum  # noqa: E402

Q_LENS = [1, 33, 1040, 1041, 1042, 2080, 2081, 4300]
Q_KINDS = ["pos", "neg", "alt", "pair"]
I8_SCALE = 1.0 / (127.0 * 127.0)
B1_SCALE = 1.0 / 128.0
ALT = np.where(np.arange(128) % 2, -127, 127)  # the sign pattern of an "alt" query
# page kinds in id order: the higher page of the pair, and +127 (above the half-magnitude pages), sit at higher ids
I8_PAGES = ["empty", "half", "minus", "alt", "pair_lo", "pair_hi", "plus", "empty", "mixed", "half", "plus"] * 6
B1_PAGES = ["empty", "zeros", "alt", "ones", "mixed", "ones", "empty", "zeros"] * 6


def vp(t):
    return ctypes.c_void_p(t.data_ptr()) if t is not None else None


def stream():
    return ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)


def bits(x):
    return np.asarray(x, np.float32).view(np.uint32)


# ------------------------------------------------------------------------------------------------ corpora and queries
def i8_rows(kind):
    full = lambda v: np.full(128, v)  # noqa: E731
    pair = full(127)
    pair[0] = 126
    rows = {"empty": [], "half": [full(64)] * 3, "minus": [full(-127)] * 2, "alt": [ALT, -ALT], "pair_lo": [pair],
            "pair_hi": [full(64), full(127)], "plus": [full(64), full(127), full(-127)],
            "mixed": [full(127), full(-127), ALT], "m128": [full(-128), full(-128)]}[kind]
    return np.asarray(rows, np.int64).reshape(-1, 128).astype(np.int8)


def b1_rows(kind):
    rows = {"empty": [], "zeros": [0x00] * 2, "ones": [0xFF], "alt": [0xAA], "mixed": [0x00, 0xAA, 0xFF, 0x0F]}[kind]
    return np.repeat(np.asarray(rows, np.uint8)[:, None], 16, axis=1)


def query(kind, t):
    q = np.ones((t, 128), np.float32)
    if kind == "neg":
        q = -q
    elif kind == "alt":
        q[:, 1::2] = -1.0
    elif kind == "pair":  # only token 0's element 0 (code 1) tells pair_lo (126 there) from pair_hi (127)
        q[:, 0] = 0.0
        q[0, 0] = 1.0 / 127.0
    return q


QUERIES = [query(kind, t) for kind in Q_KINDS for t in Q_LENS]
LENS = [len(q) for q in QUERIES]


def pad_pages(rows, lens):
    """Packed true rows [sum len, row bytes] -> the corpus layout: each page padded to 32 rows with its last row."""
    out, o = [], 0
    for n in lens:
        page = rows[o:o + n]
        o += n
        if n:
            out.append(np.concatenate([page, np.repeat(page[-1:], -n % 32, axis=0)]))
    return np.concatenate(out)


class Corpus:
    def __init__(self, dtype, kinds, rows_of):
        self.dtype, self.kinds = dtype, list(kinds)
        pages = [rows_of(k) for k in self.kinds]
        self.lens = [len(p) for p in pages]
        self.rows = np.concatenate(pages)
        self.off = orc.page_offsets(self.lens)
        self.n_pages = len(pages)
        self.scale = I8_SCALE if dtype == "int8" else B1_SCALE

    def index(self, tier="hbm", **options):
        idx = MaxSimIndex(dtype=self.dtype, tier=tier)
        for name, value in options.items():
            idx.set_option(name, value)
        packed = pad_pages(self.rows.view(np.uint8), self.lens)
        idx.append_packed(torch.from_numpy(np.ascontiguousarray(packed)).cuda(), self.lens)
        return idx

    def sums(self, queries):
        """Exact int64 sums [n_q, n_pages] of the oracle."""
        if self.dtype == "int8":
            return np.stack([orc.int8_maxsim_c(orc.quantize_int8_np(q, 127.0), self.rows, self.off) for q in queries])
        return np.stack([orc.binary_maxsim_c(orc.sign_pack_c(q), self.rows, self.off)[1] for q in queries])


@functools.lru_cache(maxsize=None)
def i8_corpus():
    return Corpus("int8", I8_PAGES, i8_rows)


@functools.lru_cache(maxsize=None)
def i8_sums():
    return i8_corpus().sums(QUERIES)


@functools.lru_cache(maxsize=None)
def i8_index(tier="hbm"):
    return i8_corpus().index(tier)


def q_dev(queries=QUERIES):
    return torch.from_numpy(np.concatenate(queries)).cuda()


def host(ts):
    return tuple(t.cpu().numpy() for t in ts)


# ------------------------------------------------------------------------------------------------ checks
def check_pages(ts, ti, tc, sums, k, scale, allow=None, id_base=0, what=""):
    """One query's top-k pages against the clamped oracle sums [n_pages]: ids, count and score bits exactly."""
    ws, wi = orc.topk_np(i32_sum(sums), k, allow)
    n = len(wi)
    assert int(tc) == n, (what, int(tc), n)
    bad = np.flatnonzero(ti[:n] != wi + id_base)
    assert not len(bad), (what, bad[:5], ti[:n][bad[:5]], wi[bad[:5]], sums[wi[bad[:5]]])
    assert np.all(ti[n:] == -1), what
    bad = np.flatnonzero(bits(ts[:n]) != bits(i32_reported(ws, scale)))
    assert not len(bad), (what, bad[:5], ts[:n][bad[:5]], i32_reported(ws, scale)[bad[:5]])


def slot_sums(sums, cand):
    valid = (cand >= 0) & (cand < len(sums))
    return np.where(valid, sums[np.where(valid, cand, 0)], 0), valid


def check_slots(ts, ti, tc, sums, cand, k, scale, what=""):
    """One query's rerank over its candidate slots: (clamped sum DESC, slot ASC), reported as page ids."""
    s, valid = slot_sums(sums, np.asarray(cand))
    ws, slots = orc.topk_np(i32_sum(s), k, valid)
    n = len(slots)
    assert int(tc) == n, (what, int(tc), n)
    bad = np.flatnonzero(ti[:n] != cand[slots])
    assert not len(bad), (what, bad[:5], ti[:n][bad[:5]], cand[slots][bad[:5]])
    assert np.all(ti[n:] == -1), what
    assert np.array_equal(bits(ts[:n]), bits(i32_reported(ws, scale))), what


def what_q(i):
    return f"q{i} {Q_KINDS[i // len(Q_LENS)]} x {LENS[i]}"


def test_the_corpus_reaches_the_limits():
    """The oracle sums cross the bound on both sides, the pair differs by 1 above 2^24 where float32 merges it, and the
    1040-token sum stays inside."""
    s = i8_sums()
    k = I8_PAGES.index
    pos = Q_KINDS.index("pos") * len(Q_LENS)
    assert s[pos + Q_LENS.index(1040), k("plus")] == 1040 * 2_064_512 <= I32_SUM_BOUND
    assert s[pos + Q_LENS.index(1041), k("plus")] > I32_SUM_BOUND and s[pos + Q_LENS.index(1041), k("minus")] < -I32_SUM_BOUND
    assert s[pos + Q_LENS.index(2081), k("half")] > I32_SUM_BOUND
    pair = Q_KINDS.index("pair") * len(Q_LENS)
    for t in range(len(Q_LENS)):
        hi, lo = s[pair + t, k("pair_hi")], s[pair + t, k("pair_lo")]
        assert hi - lo == 1
        if 1 << 24 < hi <= I32_SUM_BOUND:
            assert np.float32(hi) == np.float32(lo)
    # an int32 accumulator would rank the +127 page last and the -127 page first for 1041 tokens
    wrapped = s[pos + Q_LENS.index(1041)].astype(np.int32)
    assert wrapped[k("plus")] < 0 < wrapped[k("minus")]


# ------------------------------------------------------------------------------------------------ b200ms_score + b200ms_topk
def topk_raw(h, gs, goff, n_pages, k, scale, id_base=0):
    n_q = len(goff) - 1
    ts = torch.full((n_q, k), 7.0, dtype=torch.float32, device="cuda")
    ti = torch.full((n_q, k), -7, dtype=torch.int64, device="cuda")
    tc = torch.full((n_q,), -7, dtype=torch.int32, device="cuda")
    h.check(nat.lib.b200ms_topk(h.ptr, vp(gs), nat.I32, n_pages, gs.shape[1], nat.i32_array([int(x) for x in goff]), n_q,
                                None, k, ctypes.c_float(scale), id_base, vp(ts), vp(ti), vp(tc), stream()),
            "b200ms_topk")
    torch.cuda.synchronize()
    return host((ts, ti, tc))


M = I32_SUM_BOUND
INT_MIN = -(1 << 31)
# (4 group scores) of page p: sums M - 2, M - 1, M, M + 1, 4M, -M + 1, -M, -M - 1, 4 INT_MIN and 0.  The pages at the bound
# (2, 3, 4) tie there and come before page 1 (M - 1), which float32 reports as the same score.
BOUND_PAGES = np.asarray([[M - 2, 0, 0, 0], [M - 3, 1, 1, 0], [M - 3, 1, 1, 1], [M, 1, 0, 0], [M, M, M, M],
                          [-M + 1, 0, 0, 0], [INT_MIN, 1, 0, 0], [INT_MIN, 0, 0, 0], [INT_MIN] * 4, [M, INT_MIN, 1, 0]],
                         np.int64)


@pytest.mark.parametrize("n_pages", [10, 1030, 20000])
def test_topk_and_topk_docs_at_the_bound(n_pages):
    """b200ms_topk and b200ms_topk_docs on group scores summing to either side of the bound, the pattern repeated over
    n_pages (the counting kernel, the radix select, the sliced select)."""
    sums = np.tile(BOUND_PAGES.sum(axis=1), -(-n_pages // 10))[:n_pages]
    assert orc.topk_np(i32_sum(sums[:10]), 10)[1].tolist() == [2, 3, 4, 1, 0, 9, 5, 6, 7, 8]
    gs = np.zeros((4, n_pages + 22), np.int32)
    gs[:, :n_pages] = np.tile(BOUND_PAGES.T, (1, -(-n_pages // 10)))[:, :n_pages]
    gs = torch.from_numpy(gs).cuda()
    h = nat.Handle(0)
    k = min(n_pages, 4096)
    ts, ti, tc = topk_raw(h, gs, [0, 4], n_pages, k, 1.0)
    check_pages(ts[0], ti[0], tc[0], sums, k, 1.0, what=f"b200ms_topk n_pages={n_pages}")
    page_doc = (np.arange(n_pages) // 2).astype(np.int32)
    n_docs = int(page_doc[-1]) + 1
    kd, per_doc = min(n_docs, 1000), 2
    out = [torch.empty(shape, dtype=dt, device="cuda") for shape, dt in (((1, kd, per_doc), torch.float32),
                                                                        ((1, kd, per_doc), torch.int64),
                                                                        ((1, kd), torch.int32), ((1,), torch.int32))]
    h.check(nat.lib.b200ms_topk_docs(h.ptr, vp(gs), nat.I32, n_pages, gs.shape[1], nat.i32_array([0, 4]), 1, None,
                                     vp(torch.from_numpy(page_doc).cuda()), n_docs, kd, per_doc, ctypes.c_float(1.0), 0,
                                     *(vp(t) for t in out), stream()), "b200ms_topk_docs")
    torch.cuda.synchronize()
    scores, ids, pcounts, dcounts = host(out)
    _, wids, wcounts, nd = topk_docs_np(i32_sum(sums), page_doc, n_docs, kd, per_doc)
    assert int(dcounts[0]) == nd and np.array_equal(pcounts[0], wcounts) and np.array_equal(ids[0], wids)
    ok = wids >= 0
    assert np.array_equal(bits(scores[0][ok]), bits(i32_reported(sums[wids[ok]], 1.0)))
    h.close()


@pytest.mark.parametrize("unit_rows", [0, 64])
def test_score_and_topk_launch_shapes(unit_rows):
    c = i8_corpus()
    want = i8_sums()
    idx = c.index(**({"unit_rows": unit_rows} if unit_rows else {}))
    for max_ctas in (0, 1, 3):
        idx.set_option("max_ctas", max_ctas)
        gs, goff, n_pages, _ = idx.score_groups(QUERIES)
        torch.cuda.synchronize()
        raw = gs[:, :n_pages].cpu().numpy().astype(np.int64)
        for qi in range(len(QUERIES)):
            what = f"unit_rows={unit_rows} max_ctas={max_ctas} {what_q(qi)}"
            assert np.array_equal(raw[goff[qi]:goff[qi + 1]].sum(axis=0), want[qi]), what  # group scores: exact
        for k in (1, 5, n_pages):
            ts, ti, tc = topk_raw(idx.h, gs, goff, n_pages, k, c.scale, id_base=1 << 40)
            for qi in range(len(QUERIES)):
                check_pages(ts[qi], ti[qi], tc[qi], want[qi], k, c.scale, id_base=1 << 40,
                            what=f"unit_rows={unit_rows} max_ctas={max_ctas} k={k} {what_q(qi)}")
    idx.close()


# ------------------------------------------------------------------------------------------------ the search entry points
def test_search_host_and_graph_replay():
    c, want, idx = i8_corpus(), i8_sums(), i8_index()
    one = Q_KINDS.index("neg") * len(Q_LENS) + Q_LENS.index(1041)
    for call in range(3):  # the same layout: captured on its second use, replayed on the third
        ts, ti, tc = idx.search_host([QUERIES[one]], k=c.n_pages)
        check_pages(ts[0], ti[0], tc[0], want[one], c.n_pages, c.scale, what=f"search_host call {call}")
    for call in range(3):
        ts, ti, tc = idx.search_host(QUERIES, k=9, id_base=5)
        for qi in range(len(QUERIES)):
            check_pages(ts[qi], ti[qi], tc[qi], want[qi], 9, c.scale, id_base=5, what=f"batch call {call} {what_q(qi)}")


def test_search_device_and_masks():
    c, want, idx = i8_corpus(), i8_sums(), i8_index()
    n = c.n_pages
    ts, ti, tc = host(idx.search_device(q_dev(), LENS, n))
    for qi in range(len(QUERIES)):
        check_pages(ts[qi], ti[qi], tc[qi], want[qi], n, c.scale, what=f"search_device {what_q(qi)}")
    pos = Q_KINDS.index("pos") * len(Q_LENS) + Q_LENS.index(1041)  # +127 pages above half-magnitude ones, -127 pages last
    order = [I8_PAGES[p] for p in ti[pos][:tc[pos]]]
    assert max(i for i, kind in enumerate(order) if kind == "plus") < min(i for i, kind in enumerate(order) if kind == "half")
    assert set(order[-I8_PAGES.count("minus"):]) == {"minus"}
    assert ts[pos][0] == np.float32(np.float32(2.0 ** 31) * np.float32(I8_SCALE))
    rng = np.random.default_rng(3)
    allows = [rng.random(n) < f for f in (0.3, 0.7)]
    words = torch.from_numpy(np.stack([idx.mask_from_pages(a) for a in allows]).view(np.int32)).cuda()
    index = torch.from_numpy(np.asarray([qi % 3 - 1 for qi in range(len(QUERIES))], np.int32)).cuda()
    ts, ti, tc = host(idx.search_device(q_dev(), LENS, 12, allow_mask_dev=words, mask_index_dev=index))
    for qi in range(len(QUERIES)):
        m = qi % 3 - 1
        check_pages(ts[qi], ti[qi], tc[qi], want[qi], 12, c.scale, None if m < 0 else allows[m], what=f"masked {what_q(qi)}")
    ts, ti, tc = host(idx.search_device(q_dev(), LENS, n, allow_mask_dev=words[1]))
    for qi in range(len(QUERIES)):
        check_pages(ts[qi], ti[qi], tc[qi], want[qi], n, c.scale, allows[1], what=f"one mask {what_q(qi)}")


def test_filtered_scan():
    """Per-query masks on a corpus of several waves of work units: the masks build the scan's work units."""
    c, want = i8_corpus(), i8_sums()
    idx = c.index(unit_rows=64)
    idx.set_option("max_ctas", 3)
    rng = np.random.default_rng(4)
    allows = [rng.random(c.n_pages) < f for f in (0.2, 0.5)]
    masks = [allows[qi % 2] for qi in range(len(QUERIES))]
    ts, ti, tc = idx.search_host_masked(QUERIES, c.n_pages, [idx.mask_from_pages(m) for m in masks])
    assert 0 < idx.scan_stats()["rows"] < idx.n_rows_padded
    for qi in range(len(QUERIES)):
        check_pages(ts[qi], ti[qi], tc[qi], want[qi], c.n_pages, c.scale, masks[qi], what=f"filtered {what_q(qi)}")
    idx.close()


# ------------------------------------------------------------------------------------------------ reranks
def candidate_lists(n_pages, n_q, n_cand, seed):
    rng = np.random.default_rng(seed)
    cand = rng.integers(0, n_pages, size=(n_q, n_cand)).astype(np.int64)  # repeated pages: ties broken by slot
    cand[:, 3] = -1
    cand[:, 6] = n_pages + 9
    return cand


@pytest.mark.parametrize("n_cand,k", [(48, 7), (48, 48), (4096, 5)])
def test_reranks(n_cand, k):
    """Shared and per-query lists on both tiers (host == HBM bit for bit); 4096 candidates select through the sliced top-k."""
    c, want = i8_corpus(), i8_sums()
    cand = candidate_lists(c.n_pages, len(QUERIES), n_cand, n_cand + k)
    cd = torch.from_numpy(cand).cuda()
    out = {}
    for tier in ("hbm", "host"):
        idx = i8_index(tier)
        per_q = host(idx.rerank_batch(q_dev(), LENS, cd, k))
        shared = host(idx.rerank(q_dev(), LENS, cd[0].contiguous(), k))
        for qi in range(len(QUERIES)):
            check_slots(*(x[qi] for x in per_q), want[qi], cand[qi], k, c.scale, f"{tier} rerank_batch {what_q(qi)}")
            check_slots(*(x[qi] for x in shared), want[qi], cand[0], k, c.scale, f"{tier} rerank {what_q(qi)}")
        out[tier] = per_q + shared
    for a, b in zip(out["hbm"], out["host"]):
        assert np.array_equal(np.asarray(a).view(np.uint8), np.asarray(b).view(np.uint8))


def explain_raw(idx, queries, cand):
    """Explain's token values with score_scale 1: the integer dot products themselves (exact in float32 below 2^24)."""
    idx._attach()
    src, src_dtype = idx._stage_rows(list(queries))
    lens = [len(q) for q in queries]
    ids = torch.from_numpy(np.ascontiguousarray(cand, np.int64)).cuda()
    n_q, n_cand = ids.shape
    ts = torch.empty((n_q, n_cand, max(lens)), dtype=torch.float32, device="cuda")
    br = torch.empty((n_q, n_cand, max(lens)), dtype=torch.int32, device="cuda")
    idx.h.check(nat.lib.b200ms_explain_device(idx.h.ptr, vp(src), src_dtype, nat.i32_array(lens), n_q, vp(ids), n_cand,
                                              ctypes.c_float(idx.i8_scale), ctypes.c_float(1.0), vp(ts), vp(br), None, 0,
                                              stream()), "b200ms_explain_device")
    torch.cuda.synchronize()
    return ts.cpu().numpy(), br.cpu().numpy()


def check_explain(idx, c, queries, sums, what):
    """Every page of the corpus for every query: the integer token values sum in int64 to the oracle's exact sum, and the
    rerank of the same list reports the clamped sum."""
    cand = np.tile(np.arange(c.n_pages, dtype=np.int64), (len(queries), 1))
    tok, _ = explain_raw(idx, queries, cand)
    assert np.array_equal(tok, np.rint(tok)) and np.abs(tok).max() < 1 << 24
    got = tok.astype(np.int64).sum(axis=2)
    bad = np.argwhere(got != sums)
    assert not len(bad), (what, bad[:5], got[tuple(bad[0])], sums[tuple(bad[0])])
    lens = [len(q) for q in queries]
    ts, ti, tc = host(idx.rerank_batch(q_dev(queries), lens, torch.from_numpy(cand).cuda(), c.n_pages))
    for qi in range(len(queries)):
        check_slots(ts[qi], ti[qi], tc[qi], sums[qi], cand[qi], c.n_pages, c.scale, f"{what} rerank q{qi} x {lens[qi]}")
    return tok


def test_explain_on_both_tiers():
    c, want = i8_corpus(), i8_sums()
    toks = [check_explain(i8_index(tier), c, QUERIES, want, f"int8 {tier}") for tier in ("hbm", "host")]
    assert np.array_equal(toks[0].view(np.uint32), toks[1].view(np.uint32))  # host tier == HBM, bit for bit


# ------------------------------------------------------------------------------------------------ more than 16384 pages
def test_full_scan_over_20000_one_row_pages():
    """One-row pages of the distinct row kinds: above 2 * 8192 pages the full-scan top-k selects per slice and merges."""
    rng = np.random.default_rng(11)
    base = ["half", "minus", "alt", "pair_lo", "plus", "m128"]
    distinct = np.concatenate([i8_rows(k)[-1:] for k in base] + [i8_rows("pair_hi")[1:]])
    kinds = rng.integers(0, len(distinct), size=20000)
    c = Corpus("int8", list(kinds), lambda k: distinct[k:k + 1])
    pick = [Q_KINDS.index(kind) * len(Q_LENS) + Q_LENS.index(t) for kind in ("pos", "neg", "pair") for t in (1040, 1041, 2081)]
    qs = [QUERIES[i] for i in pick]
    per_row = Corpus("int8", range(len(distinct)), lambda k: distinct[k:k + 1]).sums(qs)
    want = per_row[:, kinds]
    idx = c.index()
    for k in (10, 1000):
        ts, ti, tc = host(idx.search_device(q_dev(qs), [len(q) for q in qs], k))
        for qi in range(len(qs)):
            check_pages(ts[qi], ti[qi], tc[qi], want[qi], k, c.scale, what=f"20000 pages k={k} {what_q(pick[qi])}")
    idx.close()


# ------------------------------------------------------------------------------------------------ documents
def test_document_searches():
    c, want, idx = i8_corpus(), i8_sums(), i8_index()
    page_doc = (np.arange(c.n_pages) // 3).astype(np.int32)
    n_docs = int(page_doc.max()) + 1
    pd = torch.from_numpy(page_doc).cuda()
    k, per_doc = 9, 2
    scores, ids, pcounts, dcounts = idx.search_docs(QUERIES, k, per_doc, pd, n_docs)
    for qi in range(len(QUERIES)):
        _, wids, wcounts, nd = topk_docs_np(i32_sum(want[qi]), page_doc, n_docs, k, per_doc)
        what = f"search_docs {what_q(qi)}"
        assert int(dcounts[qi]) == nd and np.array_equal(pcounts[qi], wcounts) and np.array_equal(ids[qi], wids), what
        ok = wids >= 0
        assert np.array_equal(bits(scores[qi][ok]), bits(i32_reported(want[qi][wids[ok]], c.scale))), what
    cand = candidate_lists(c.n_pages, len(QUERIES), 64, 13)
    out = idx.rerank_docs_batch(q_dev(), LENS, torch.from_numpy(cand).cuda(), k, per_doc, pd, n_docs)
    scores, ids, pcounts, dcounts = host(out)
    for qi in range(len(QUERIES)):
        s, _ = slot_sums(want[qi], cand[qi])
        _, wids, wcounts, nd = topk_docs_np(i32_sum(s), page_doc, n_docs, k, per_doc, cand=cand[qi])
        what = f"rerank_docs {what_q(qi)}"
        assert int(dcounts[qi]) == nd and np.array_equal(pcounts[qi], wcounts) and np.array_equal(ids[qi], wids), what
        ok = wids >= 0
        assert np.array_equal(bits(scores[qi][ok]), bits(i32_reported(want[qi][wids[ok]], c.scale))), what


# ------------------------------------------------------------------------------------------------ the sign first stage
def test_sign_stage_into_int8_rerank():
    """Every page is a candidate; the rerank orders them by the clamped sum, ties by the first stage's rank (slot)."""
    c, want = i8_corpus(), i8_sums()
    sti = SignTwoStageIndex(dtype="int8")
    packed = pad_pages(c.rows.view(np.uint8), c.lens)
    sti.index.append_packed(torch.from_numpy(np.ascontiguousarray(packed)).cuda(), c.lens)
    sti.rebuild_from_index()
    ci, _, cc = host(sti.candidates(QUERIES, c.n_pages))
    assert np.all(cc > 0)
    ts, ti, tc, _ = sti.search_device(QUERIES, k=20, n_candidates=c.n_pages)
    ts, ti, tc = host((ts, ti, tc))
    for qi in range(len(QUERIES)):
        check_slots(ts[qi], ti[qi], tc[qi], want[qi], ci[qi], 20, c.scale, f"two-stage {what_q(qi)}")


# ------------------------------------------------------------------------------------------------ -128 rows
def test_minus_128_rows_reach_the_bound_at_1033_tokens():
    """A -1.0 query (codes -127) scores 128 * 127 * 128 per token against a row of -128."""
    c = Corpus("int8", ["m128", "plus", "minus", "empty", "half", "m128"], i8_rows)
    qs = [-np.ones((t, 128), np.float32) for t in (1, 1032, 1033, 2065)]
    want = c.sums(qs)
    assert want[1, 0] == 1032 * 2_080_768 <= I32_SUM_BOUND < want[2, 0]
    idx = c.index()
    lens = [len(q) for q in qs]
    ts, ti, tc = host(idx.search_device(q_dev(qs), lens, c.n_pages))
    for qi in range(len(qs)):
        check_pages(ts[qi], ti[qi], tc[qi], want[qi], c.n_pages, c.scale, what=f"-128 search_device x {lens[qi]}")
    check_explain(idx, c, qs, want, "-128")
    idx.close()


# ------------------------------------------------------------------------------------------------ 1-bit
@functools.lru_cache(maxsize=None)
def b1_corpus():
    return Corpus("binary", B1_PAGES, b1_rows)


@pytest.mark.parametrize("b1_tensor", [0, 1])
def test_binary_long_queries(b1_tensor):
    """POPC (0) and wgmma with bit expansion (1) full scans, the rerank and explain, exact against the oracle."""
    c = b1_corpus()
    qs = [q for q, kind in zip(QUERIES, [k for k in Q_KINDS for _ in Q_LENS]) if kind != "pair"]
    want = c.sums(qs)
    assert want.max() == 4300 * 128  # far below the bound: no clamping
    idx = c.index(b1_tensor=b1_tensor)
    lens = [len(q) for q in qs]
    gs, goff, n_pages, _ = idx.score_groups(qs)
    torch.cuda.synchronize()
    raw = gs[:, :n_pages].cpu().numpy().astype(np.int64)
    for qi in range(len(qs)):
        assert np.array_equal(raw[goff[qi]:goff[qi + 1]].sum(axis=0), want[qi]), (b1_tensor, qi, lens[qi])
    ts, ti, tc = idx.search_host(qs, k=c.n_pages)
    for qi in range(len(qs)):
        check_pages(ts[qi], ti[qi], tc[qi], want[qi], c.n_pages, c.scale, what=f"b1_tensor={b1_tensor} q{qi} x {lens[qi]}")
    check_explain(idx, c, qs, want, f"b1_tensor={b1_tensor}")
    idx.close()


# ------------------------------------------------------------------------------------------------ the store
def test_store_ranks_the_plus_page_first_at_1041_tokens():
    store = B200MultiVectorStore(mode="int8")
    pages = {"minus": -np.ones((3, 128), np.float32), "half": np.full((2, 128), 0.5, np.float32),
             "plus": np.ones((4, 128), np.float32), "empty_ish": np.zeros((1, 128), np.float32)}
    chunks = [DocumentChunk(document_id=name, chunk_number=0, content=name, metadata={}, embedding=e) for name, e in pages.items()]
    asyncio.run(store.store_embeddings(chunks))
    q = np.ones((1041, 128), np.float32)
    got = asyncio.run(store.query_similar(q, k=4))
    rows = np.concatenate(list(pages.values()))
    sums = orc.int8_maxsim_c(orc.quantize_int8_np(q, 127.0), orc.quantize_int8_np(rows, 127.0),
                             orc.page_offsets([len(p) for p in pages.values()]))
    order = np.argsort(-i32_sum(sums), kind="stable")
    assert [c.document_id for c in got] == [list(pages)[i] for i in order]
    assert got[0].document_id == "plus" and got[-1].document_id == "minus"
    assert [np.float32(c.score) for c in got] == list(i32_reported(sums[order], I8_SCALE))
    assert np.float32(got[0].score) == np.float32(np.float32(2.0 ** 31) * np.float32(I8_SCALE))
    store.close()
