"""The bf16 and fp8 scorers on every input value, infinities and NaNs included (run with -m gpu on an H100).

The expected values come from tests/float_value_oracle.py, the float value rule of include/b200ms.h in float64.  Comparisons
are exact where the rule leaves nothing to rounding: NaN must be NaN, +-inf the same infinity, and a probe score (one nonzero
product) its exact value.  Finite scores of the mixed corpora keep oracle.scoring.TOL.

  * Probes: single-row pages holding every bf16 pattern (every e4m3 code), read out by one-hot one-token queries, so
    score[q_i, p] = row_p[i]; pairs of powers of two whose product overflows, lands in fp32's subnormal range or underflows.
  * Non-finite corpora: +-inf or NaN in one row, in every row, with mixed signs across rows, and +inf meeting -inf inside a
    row; queries of 1, 31, 32, 33, 64 and 65 tokens meet those elements with 0, a positive and a negative value, so a query's
    last group has padding tokens or none.  A zero padding token meets 0 * inf = NaN on a page whose rows all hold an infinity:
    only the true tokens may count.
  * Every path that scores these corpora: the full scan (NM 1 / 2 / 4, split CTA pairs, max_ctas 0 / 1 / 3, unit_rows default /
    64), the filtered scan, search_host (graph replay included), search_device, both reranks, search_docs and rerank_docs,
    explain (its token scores add up to the rerank's score), the host tier's reranks and explain, and zero_pad_compat.
"""
import functools

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

torch = pytest.importorskip("torch")
if not torch.cuda.is_available():  # pragma: no cover - the gpu marker normally deselects these on CPU boxes
    pytest.skip("CUDA device required", allow_module_level=True)

import float_value_oracle as fvo  # noqa: E402
from docs_oracle import topk_docs_np  # noqa: E402
from morphik_core_b200.index import MaxSimIndex  # noqa: E402
from oracle import maxsim_oracle as orc  # noqa: E402
from oracle.scoring import TOL  # noqa: E402

DTYPES = ["bf16", "fp8"]
UNIT = {"bf16": 1.0, "fp8": fvo.F8_SCALE ** 2}  # packed units per reference-scale unit
INF, NAN = np.inf, np.nan


def same_values(got, want, tol=0.0):
    """Mismatches of got against want: NaN only against NaN, +-inf only against the same infinity, finite values equal
    (tol = 0; +-0 alike) or within tol relative (floor 1e-3).  Returns the indices that differ."""
    got, want = np.asarray(got, np.float64), np.asarray(want, np.float64)
    fin = np.isfinite(want)
    with np.errstate(invalid="ignore"):
        bad = ~fin & ~((np.isnan(got) & np.isnan(want)) | (got == want))
        err = np.abs(got - want) / np.maximum(np.abs(want), 1e-3)
    bad |= fin & ~(np.isfinite(got) & (err <= tol))
    return np.argwhere(bad)


def assert_values(got, want, tol, what, labels=None):
    bad = same_values(got, want, tol)
    if len(bad):
        first = [(tuple(int(i) for i in b), float(np.asarray(got)[tuple(b)]), float(np.asarray(want)[tuple(b)]))
                 for b in bad[:6]]
        raise AssertionError(f"{what}: {len(bad)} of {np.asarray(want).size} differ, first {first}"
                             + (f" ({labels(bad)})" if labels else ""))


def pad_pages(rows: np.ndarray, lens):
    """Packed true rows [sum len, row bytes] -> the padded corpus layout (a page's last row repeated to 32 rows)."""
    out, o = [], 0
    for n in lens:
        page = rows[o:o + n]
        o += n
        if n:
            out.append(np.concatenate([page, np.repeat(page[-1:], -n % 32, axis=0)]))
    return np.concatenate(out)


def packed_index(dtype, rows_u8, lens):
    idx = MaxSimIndex(dtype=dtype)
    idx.append_packed(torch.from_numpy(np.ascontiguousarray(pad_pages(rows_u8, lens))).cuda(), lens)
    return idx


def one_hot_queries(n, value=1.0):
    qs = []
    for i in range(n):
        q = np.zeros((1, 128), np.float32)
        q[0, i % 128] = value
        qs.append(q)
    return qs


# ------------------------------------------------------------------------------------------------ a. probes
def bf16_probe_rows():
    """Every finite bf16 pattern, 128 to a row, then one row per non-finite pattern (at position j % 128, zeros elsewhere)."""
    pats = np.arange(65536, dtype=np.uint32).astype(np.uint16)
    nonfin = (pats & 0x7F80) == 0x7F80
    fin_rows = pats[~nonfin].reshape(-1, 128)
    nf = pats[nonfin]
    nf_rows = np.zeros((len(nf), 128), np.uint16)
    nf_rows[np.arange(len(nf)), np.arange(len(nf)) % 128] = nf
    return np.concatenate([fin_rows, nf_rows])


def probe_scores(dtype, idx, qs):
    return idx.score_matrix(qs) * UNIT[dtype]


def expected_one_row_pages(q_vals, d_vals):
    """Scores of one-token queries on one-row pages: the similarity itself (one token, one row)."""
    return np.concatenate([fvo.similarities(q_vals, d_vals[i:i + 64]) for i in range(0, len(d_vals), 64)], axis=1)


def test_bf16_probe_every_pattern():
    rows = bf16_probe_rows()                                     # [766, 128] patterns
    idx = packed_index("bf16", rows.view(np.uint8).reshape(len(rows), 256), [1] * len(rows))
    qs = one_hot_queries(128)
    got = probe_scores("bf16", idx, qs)
    want = expected_one_row_pages(fvo.pack_values("bf16", np.concatenate(qs)), fvo.bf16_values(rows))
    # finite rows: score[q_i, p] = row_p[i] exactly, subnormal patterns included
    fin = rows[:510]
    assert np.array_equal(want[:, :510], fvo.bf16_values(fin).T)
    sub = (fin.T & 0x7F80) == 0

    def labels(bad):
        return f"{int(sum(1 for i, p in bad if p < 510 and sub[i, p]))} of them subnormal patterns"
    assert_values(got, want, 0.0, "bf16 probes", labels)
    nz = np.isfinite(want) & (want != 0)
    assert np.array_equal(got[nz].astype(np.float32).view(np.uint32), want[nz].astype(np.float32).view(np.uint32))


def test_fp8_probe_every_code():
    codes = np.arange(256, dtype=np.uint8)
    nan = (codes & 0x7F) == 0x7F
    fin = np.concatenate([codes[~nan], np.zeros(2, np.uint8)]).reshape(2, 128)
    nf = np.zeros((2, 128), np.uint8)
    nf[0, 3], nf[1, 100] = 0x7F, 0xFF
    rows = np.concatenate([fin, nf])
    idx = packed_index("fp8", rows, [1] * len(rows))
    qs = one_hot_queries(128)
    got = probe_scores("fp8", idx, qs)
    qv = fvo.pack_values("fp8", np.concatenate(qs))
    assert np.all(qv.max(axis=1) == 64.0)  # 1.0 * 64 is the e4m3 code of 64
    want = expected_one_row_pages(qv, fvo.e4m3_values(rows))
    assert np.array_equal(want[:, :2], 64.0 * fvo.e4m3_values(fin).T)
    assert np.isnan(want[:, 2:]).all()
    assert_values(got, want, 0.0, "fp8 probes")


# (query exponent, row exponent, sign): one-token queries against one-row pages at position i
PRODUCT_PAIRS = [(64, 64, 1), (64, 64, -1), (63, 64, 1), (127, 1, 1), (127, 127, 1), (-63, -64, 1), (-63, -64, -1),
                 (-70, -70, 1), (-70, -79, 1), (-75, -75, 1), (-100, -100, 1), (-133, 0, 1), (-133, -1, 1), (-126, -1, 1)]


def test_bf16_products_leave_the_fp32_range():
    qs, pages = [], []
    for i, (a, b, sgn) in enumerate(PRODUCT_PAIRS):
        q = np.zeros((1, 128), np.float32)
        d = np.zeros((1, 128), np.float32)
        q[0, i], d[0, i] = sgn * 2.0 ** a, 2.0 ** b
        qs.append(q)
        pages.append(d)
    # two products past fp32's range that cancel (one MMA step); a finite sum past the fp32 range
    q = np.zeros((1, 128), np.float32)
    d = np.zeros((1, 128), np.float32)
    q[0, 20:22], d[0, 20:22] = [2.0 ** 64, -(2.0 ** 64)], 2.0 ** 64
    qs.append(q)
    pages.append(d)
    q = np.zeros((1, 128), np.float32)
    d = np.zeros((1, 128), np.float32)
    q[0, 30:32], d[0, 30:32] = 1.0, 2.0 ** 127
    qs.append(q)
    pages.append(d)
    idx = MaxSimIndex(dtype="bf16")
    idx.add_pages(pages)
    got = idx.score_matrix(qs)
    qv, dv = fvo.pack_values("bf16", np.concatenate(qs)), fvo.pack_values("bf16", np.concatenate(pages))
    want = expected_one_row_pages(qv, dv)
    diag = np.diag(want)
    assert diag[0] == INF and diag[1] == -INF and diag[5] == 2.0 ** -127 and diag[8] == 2.0 ** -149 and diag[9] == 0.0
    assert diag[-2] == 0.0 and diag[-1] == INF
    assert_values(got, want, 0.0, f"bf16 products {list(zip(PRODUCT_PAIRS, np.diag(got)))}")


# ------------------------------------------------------------------------------------------------ b. non-finite corpora
J0, J1, J2 = 5, 77, 126  # elements that hold the infinities (J0, J2) and the NaNs (J1)
PAGE_KINDS = ["finite", "inf_one_row", "inf_every_row", "neginf_every_row", "inf_mixed_signs", "nan_one_row",
              "nan_every_row", "nan_and_inf_rows", "inf_cancel_in_row", "empty"]
PAGE_LENS = [1, 31, 33, 64, 65]
Q_LENS = [1, 31, 32, 33, 64, 65]
Q_KINDS = ["pos", "neg", "zero", "mixed"]


@functools.lru_cache(maxsize=None)
def special_corpus():
    """(pages float32, kinds): every page kind at every length (an empty page once), twice over."""
    rng = np.random.default_rng(2026)
    pages, kinds = [], []
    for rep in range(2):
        for kind in PAGE_KINDS:
            for n in ([0] if kind == "empty" else PAGE_LENS):
                d = (rng.standard_normal((n, 128)) / np.sqrt(128)).astype(np.float32)
                d[:, [J0, J1, J2]] = 0.25
                r = rng.integers(0, max(n, 1))
                if kind == "inf_one_row":
                    d[r, J0] = INF
                elif kind == "inf_every_row":
                    d[:, J0] = INF
                elif kind == "neginf_every_row":
                    d[:, J0] = -INF
                elif kind == "inf_mixed_signs":
                    d[:, J0] = np.where(np.arange(n) % 2, INF, -INF)
                elif kind == "nan_one_row":
                    d[r, J1] = NAN
                elif kind == "nan_every_row":
                    d[:, J1] = NAN
                elif kind == "nan_and_inf_rows":
                    d[:, J0] = INF
                    d[::2, J1] = NAN
                elif kind == "inf_cancel_in_row":
                    d[:, J0], d[:, J2] = INF, -INF
                    d[-1, J2] = 0.5  # one row without the cancellation
                pages.append(d)
                kinds.append(kind)
    return pages, kinds


@functools.lru_cache(maxsize=None)
def special_queries():
    """One query per (kind, length): element J0 of every token is 0 (zero), > 0 (pos), < 0 (neg) or cycles (mixed)."""
    rng = np.random.default_rng(7)
    qs = []
    for kind in Q_KINDS:
        for t in Q_LENS:
            q = (rng.standard_normal((t, 128)) / np.sqrt(128)).astype(np.float32)
            mag = np.abs(q[:, J0]) + 0.125
            sel = {"pos": np.ones(t), "neg": -np.ones(t), "zero": np.zeros(t), "mixed": np.array([1, -1, 0])[np.arange(t) % 3]}
            q[:, J0] = mag * sel[kind]
            q[:, J2] = 0.25 * (np.arange(t) % 2)  # meets the -inf of inf_cancel_in_row with 0 and with 0.25
            qs.append(q)
    return qs


@functools.lru_cache(maxsize=None)
def expected(dtype, src="f32", clamp_batch=0, page_src=None):
    """Oracle scores [n_q, n_pages] on the reference scale (what score_matrix and the top-k report) for queries from `src`
    and pages from `page_src` (default: the same)."""
    pages, _ = special_corpus()
    qs = special_queries()
    if src == "bf16":  # a bf16 source is widened exactly, then packed
        qs = [orc.bf16_round_np(q) for q in qs]
    if (page_src or src) == "bf16":
        pages = [orc.bf16_round_np(p) for p in pages]
    clamp = fvo.zero_pad_clamped([len(p) for p in pages], clamp_batch) if clamp_batch else None
    qv = [fvo.pack_values(dtype, q) for q in qs]
    dv = [fvo.pack_values(dtype, p) for p in pages]
    return fvo.scores(qv, dv, clamp) / UNIT[dtype]


def to_source(x, src):
    t = torch.from_numpy(np.ascontiguousarray(x)).cuda()
    return t.to(torch.bfloat16) if src == "bf16" else t


@functools.lru_cache(maxsize=None)
def special_index(dtype, src="f32", tier="hbm"):
    pages, _ = special_corpus()
    idx = MaxSimIndex(dtype=dtype, tier=tier)
    idx.add_pages([to_source(p, src) for p in pages] if src == "bf16" else pages)
    return idx


def queries_of(src):
    qs = special_queries()
    return [to_source(q, src) for q in qs] if src == "bf16" else qs


def test_the_corpus_exercises_every_outcome():
    """The oracle gives the pages NaN, +inf, -inf and finite scores, and without the padding rule (every query padded to
    whole 32-token groups with zero rows) some of them would change."""
    for dtype in DTYPES:
        want = expected(dtype)
        assert np.isnan(want).any() and np.isfinite(want).any()
        if dtype == "bf16":  # e4m3 saturates infinities to +-448
            assert (want == INF).any() and (want == -INF).any()
    pages, _ = special_corpus()
    qv = [fvo.pack_values("bf16", q) for q in special_queries()]
    padded = [np.vstack([q, np.zeros((-len(q) % 32, 128))]) for q in qv]
    dv = [fvo.pack_values("bf16", p) for p in pages]
    assert np.isnan(fvo.scores(padded, dv)).sum() > np.isnan(fvo.scores(qv, dv)).sum()


@pytest.mark.parametrize("src", ["f32", "bf16"])
@pytest.mark.parametrize("dtype", DTYPES)
def test_full_scan_launch_shapes(dtype, src):
    """NM 1 (1 tile), NM 2 (2 tiles), NM 4 with a phantom tile (3 tiles), split CTA pairs + NM 2 (10 tiles)."""
    qs, want = queries_of(src), expected(dtype, src)
    batches = {"nm1": [0], "nm2": [0, 1, 2, 3], "nm4": list(range(6)), "split": list(range(len(qs)))}
    for unit_rows in (0, 64):
        idx = MaxSimIndex(dtype=dtype)
        if unit_rows:
            idx.set_option("unit_rows", unit_rows)
        idx.add_pages([to_source(p, src) for p in special_corpus()[0]] if src == "bf16" else special_corpus()[0])
        for max_ctas in (0, 1, 3):
            idx.set_option("max_ctas", max_ctas)
            for name, sel in batches.items():
                got = idx.score_matrix([qs[i] for i in sel])
                assert_values(got, want[sel], TOL[dtype], f"{dtype} src={src} unit_rows={unit_rows} max_ctas={max_ctas} {name}")


def check_ranking(dtype, ts, ti, tc, want, k, allow=None, what=""):
    """One query's top-k in the total order: NaN first, then +inf, finite DESC, -inf last; ties by id.  Non-finite
    positions must hold exactly the oracle's ids; a finite position may hold another id only on a near-tie."""
    ws, wi = orc.topk_np(want, k, allow)
    n = len(wi)
    assert int(tc) == n, (what, int(tc), n)
    assert np.all(ti[n:] == -1), what
    assert_values(ts[:n], ws, TOL[dtype], f"{what} scores")
    tol = TOL[dtype]
    for i in range(n):
        if ti[i] == wi[i]:
            continue
        own = want[ti[i]]
        assert np.isfinite(ws[i]) and np.isfinite(own) and abs(own - ws[i]) <= 4 * tol * max(abs(ws[i]), 1e-3), \
            (what, i, int(ti[i]), int(wi[i]), own, ws[i])


def test_ranking_puts_nan_first_and_minus_inf_last():
    """The pos queries meet inf_every_row with +inf and neginf_every_row with -inf; nan_every_row is NaN for every query."""
    _, kinds = special_corpus()
    want = expected("bf16")
    idx = special_index("bf16")
    qs = special_queries()
    n_pages = len(kinds)
    ts, ti, tc = idx.search_host(qs, k=n_pages)
    for qi in range(len(qs)):
        check_ranking("bf16", ts[qi], ti[qi], tc[qi], want[qi], n_pages, what=f"q{qi}")
    pos = Q_KINDS.index("pos") * len(Q_LENS) + Q_LENS.index(33)
    order = [kinds[p] for p in ti[pos][:tc[pos]]]
    w = want[pos][ti[pos][:tc[pos]]]
    n_nan, n_inf, n_ninf = int(np.isnan(w).sum()), int(np.isposinf(w).sum()), int(np.isneginf(w).sum())
    assert np.isnan(w[:n_nan]).all() and np.isposinf(w[n_nan:n_nan + n_inf]).all() and np.isneginf(w[len(w) - n_ninf:]).all()
    assert "nan_every_row" in order[:n_nan] and "inf_every_row" in order[n_nan:n_nan + n_inf]
    assert "neginf_every_row" in order[len(order) - n_ninf:] and n_nan and n_inf and n_ninf


@pytest.mark.parametrize("dtype", DTYPES)
def test_search_paths(dtype):
    """search_host (twice more: the second and third calls replay the captured graph), search_host_masked, the filtered scan
    (max_ctas 3 makes the corpus more than one wave, so the masks build the work units), and search_device from f32 and bf16
    queries."""
    want = expected(dtype)
    n_pages = want.shape[1]
    qs = special_queries()
    rng = np.random.default_rng(5)
    allowed = rng.random(n_pages) < 0.6
    idx = special_index(dtype)
    idx.set_option("max_ctas", 0)
    one = [qs[Q_LENS.index(33)]]
    for call in range(3):  # a small unmasked search: captured on its second use, replayed on the third
        ts, ti, tc = idx.search_host(one, k=n_pages)
        check_ranking(dtype, ts[0], ti[0], tc[0], want[Q_LENS.index(33)], n_pages, what=f"{dtype} search_host call {call}")
    ts, ti, tc = idx.search_host(qs, k=20)
    for qi in range(len(qs)):
        check_ranking(dtype, ts[qi], ti[qi], tc[qi], want[qi], 20, what=f"{dtype} search_host q{qi}")
    idx.set_option("max_ctas", 3)
    try:
        masks = [None if qi % 3 == 0 else allowed if qi % 3 == 1 else ~allowed for qi in range(len(qs))]
        ts, ti, tc = idx.search_host_masked(qs, n_pages, [None if m is None else idx.mask_from_pages(m) for m in masks])
        for qi in range(len(qs)):
            check_ranking(dtype, ts[qi], ti[qi], tc[qi], want[qi], n_pages, masks[qi], f"{dtype} filtered q{qi}")
        ts, ti, tc = idx.search_host(qs, k=n_pages, allow_mask=idx.mask_from_pages(allowed))
        assert 0 < idx.scan_stats()["rows"] < idx.n_rows_padded  # the masks built the work units
        for qi in range(len(qs)):
            check_ranking(dtype, ts[qi], ti[qi], tc[qi], want[qi], n_pages, allowed, f"{dtype} one-mask q{qi}")
    finally:
        idx.set_option("max_ctas", 0)
    for src in ("f32", "bf16"):
        wsrc = expected(dtype, src, page_src="f32")
        q_dev = torch.cat(queries_of(src)) if src == "bf16" else torch.from_numpy(np.concatenate(qs)).cuda()
        ts, ti, tc = (t.cpu().numpy() for t in idx.search_device(q_dev, [len(q) for q in qs], n_pages))
        for qi in range(len(qs)):
            check_ranking(dtype, ts[qi], ti[qi], tc[qi], wsrc[qi], n_pages, what=f"{dtype} search_device {src} q{qi}")


def candidate_lists(n_pages, n_q, seed):
    rng = np.random.default_rng(seed)
    cand = np.stack([rng.permutation(n_pages) for _ in range(n_q)]).astype(np.int64)
    cand[:, 4] = -1
    cand[:, 9] = cand[:, 2]  # a page in two slots: the earlier slot ranks first on a tie
    return cand


def check_candidates(dtype, ts, ti, tc, want_q, cand, k, what):
    valid = (cand >= 0) & (cand < len(want_q))
    slot_scores = np.where(valid, want_q[np.where(valid, cand, 0)], 0.0)
    ws, slots = orc.topk_np(slot_scores, k, valid)
    n = len(slots)
    assert int(tc) == n, (what, int(tc), n)
    assert_values(ts[:n], ws, TOL[dtype], f"{what} scores")
    for i in range(n):
        if ti[i] != cand[slots[i]]:
            own = want_q[ti[i]]
            assert np.isfinite(ws[i]) and abs(own - ws[i]) <= 4 * TOL[dtype] * max(abs(ws[i]), 1e-3), (what, i)


def rerank_shared(idx, qs, cand, k):
    q_dev = torch.from_numpy(np.concatenate(qs)).cuda()
    out = idx.rerank(q_dev, [len(q) for q in qs], torch.from_numpy(cand).cuda(), k)
    return tuple(t.cpu().numpy() for t in out)


def rerank_batch(idx, qs, cand, k):
    q_dev = torch.from_numpy(np.concatenate(qs)).cuda()
    out = idx.rerank_batch(q_dev, [len(q) for q in qs], torch.from_numpy(np.ascontiguousarray(cand)).cuda(), k)
    return tuple(t.cpu().numpy() for t in out)


def explain_sums(idx, qs, cand):
    """Per (query, slot): the sum of explain's token scores (float64 IEEE sum), and the token scores themselves."""
    ts, br, _ = idx.explain(qs, torch.from_numpy(np.ascontiguousarray(cand)).cuda())
    tok = ts.cpu().numpy().astype(np.float64)
    return np.sum(tok, axis=-1), tok, br.cpu().numpy()


@pytest.mark.parametrize("tier", ["hbm", "host"])
@pytest.mark.parametrize("dtype", DTYPES)
def test_reranks_and_explain(dtype, tier):
    """Both reranks against the oracle, and explain: its token scores are the oracle's token maxima (exact where non-finite),
    zero past a query's length, and they add up to the score the rerank reports -- NaN and infinities included."""
    want = expected(dtype)
    n_q, n_pages = want.shape
    qs = special_queries()
    idx = special_index(dtype, tier=tier)
    cand = candidate_lists(n_pages, n_q, 9)
    k = n_pages
    ts, ti, tc = rerank_batch(idx, qs, cand, k)
    for qi in range(n_q):
        check_candidates(dtype, ts[qi], ti[qi], tc[qi], want[qi], cand[qi], k, f"{dtype} {tier} rerank_batch q{qi}")
    ts, ti, tc = rerank_shared(idx, qs, cand[0], k)
    for qi in range(n_q):
        check_candidates(dtype, ts[qi], ti[qi], tc[qi], want[qi], cand[0], k, f"{dtype} {tier} rerank q{qi}")
    # explain the reranked pages of every query, in the order the rerank returned them
    ts, ti, tc = rerank_batch(idx, qs, cand, k)
    sums, tok, _ = explain_sums(idx, qs, ti)
    pages, _ = special_corpus()
    for qi, q in enumerate(qs):
        qv = fvo.pack_values(dtype, q)
        n = int(tc[qi])
        assert np.all(tok[qi, :, len(q):] == 0.0), f"{dtype} {tier} explain: tokens past the query's length"
        for j in range(n):
            p = int(ti[qi, j])
            d = fvo.pack_values(dtype, pages[p])
            m = fvo.token_maxima(qv, d) / UNIT[dtype] if len(d) else np.zeros(len(q))
            assert_values(tok[qi, j, :len(q)], m, TOL[dtype], f"{dtype} {tier} explain q{qi} page {p}")
        # the token scores add up to the reported score: exactly for NaN / +-inf, up to the order of the sum otherwise
        assert_values(sums[qi, :n], ts[qi, :n], 1e-5, f"{dtype} {tier} explain sum vs rerank q{qi}")


@pytest.mark.parametrize("dtype", DTYPES)
def test_document_searches(dtype):
    """search_docs and rerank_docs group the same scores: two pages per document, per_doc 2."""
    want = expected(dtype)
    n_q, n_pages = want.shape
    qs = special_queries()
    idx = special_index(dtype)
    page_doc = np.arange(n_pages, dtype=np.int32) // 2
    n_docs = int(page_doc.max()) + 1
    pd_dev = torch.from_numpy(page_doc).cuda()
    k, per_doc = 12, 2
    scores, ids, pcounts, dcounts = idx.search_docs(qs, k, per_doc, pd_dev, n_docs)
    for qi in range(n_q):
        pos, wids, wcounts, nd = topk_docs_np(want[qi], page_doc, n_docs, k, per_doc)
        what = f"{dtype} search_docs q{qi}"
        assert int(dcounts[qi]) == nd and np.array_equal(pcounts[qi], wcounts), what
        ok = wids >= 0
        assert_values(scores[qi][ok], want[qi][wids[ok]], TOL[dtype], what)
        fin = ok & np.isfinite(want[qi][np.maximum(wids, 0)])
        assert np.array_equal(ids[qi][ok & ~fin], wids[ok & ~fin]), what  # non-finite pages: exactly the oracle's
    cand = candidate_lists(n_pages, n_q, 13)
    q_dev = torch.from_numpy(np.concatenate(qs)).cuda()
    out = idx.rerank_docs_batch(q_dev, [len(q) for q in qs], torch.from_numpy(cand).cuda(), k, per_doc, pd_dev, n_docs)
    scores, ids, pcounts, dcounts = (t.cpu().numpy() for t in out)
    for qi in range(n_q):
        valid = (cand[qi] >= 0) & (cand[qi] < n_pages)
        slot_scores = np.where(valid, want[qi][np.where(valid, cand[qi], 0)], 0.0)
        pos, wids, wcounts, nd = topk_docs_np(slot_scores, page_doc, n_docs, k, per_doc, cand=cand[qi])
        what = f"{dtype} rerank_docs q{qi}"
        assert int(dcounts[qi]) == nd and np.array_equal(pcounts[qi], wcounts), what
        ok = wids >= 0
        assert_values(scores[qi][ok], want[qi][wids[ok]], TOL[dtype], what)
        fin = ok & np.isfinite(want[qi][np.maximum(wids, 0)])
        assert np.array_equal(ids[qi][ok & ~fin], wids[ok & ~fin]), what


# ------------------------------------------------------------------------------------------------ d. zero_pad_compat
@pytest.mark.parametrize("dtype", DTYPES)
def test_zero_pad_compat_turns_nan_maxima_into_zero(dtype):
    """A clamped page's token max m becomes fmaxf(m, 0): a NaN max is 0 there, -inf is 0, +inf stays.  Full scan (pages in
    id order, batches of 7) and per-query rerank (slots in list order)."""
    batch = 7
    pages, _ = special_corpus()
    qs = special_queries()
    idx = MaxSimIndex(dtype=dtype)
    idx.set_option("zero_pad_compat", batch)
    idx.add_pages(pages)
    want = expected(dtype, "f32", batch)
    clean = expected(dtype)
    assert np.isnan(clean).sum() > np.isnan(want).sum()  # the clamp removes NaNs
    for max_ctas in (0, 3):
        idx.set_option("max_ctas", max_ctas)
        assert_values(idx.score_matrix(qs), want, TOL[dtype], f"{dtype} zero_pad full scan max_ctas={max_ctas}")
    idx.set_option("max_ctas", 0)
    n_q, n_pages = want.shape
    cand = candidate_lists(n_pages, n_q, 21)
    ts, ti, tc = rerank_batch(idx, qs, cand, n_pages)
    qv = [fvo.pack_values(dtype, q) for q in qs]
    for qi in range(n_q):
        sub = [pages[c] if 0 <= c < n_pages else np.zeros((0, 128), np.float32) for c in cand[qi]]
        clamp = fvo.zero_pad_clamped([len(p) for p in sub], batch)
        slot_want = np.array([fvo.page_score(qv[qi], fvo.pack_values(dtype, d), c) for d, c in zip(sub, clamp)]) / UNIT[dtype]
        valid = (cand[qi] >= 0) & (cand[qi] < n_pages)
        ws, slots = orc.topk_np(slot_want, n_pages, valid)
        n = len(slots)
        assert int(tc[qi]) == n
        assert_values(ts[qi][:n], ws, TOL[dtype], f"{dtype} zero_pad rerank q{qi}")
