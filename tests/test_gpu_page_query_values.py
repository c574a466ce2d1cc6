"""Stored pages as the QUERY operand on every input value (run with -m gpu on an H100): b200ms_search_pages_device,
b200ms_rerank_pages_batch_device, b200ms_page_rows_device, the example calls and b200ms_mmr_device.

A page query puts values on the scan's query side that no float query can: int8 -128 codes (the query quantiser clamps to
+-127), bf16 infinities and NaNs, every e4m3 code.  The expected values come from tests/float_value_oracle.py on the packed
bytes, with the exactness classes of test_gpu_scorer_values.py: NaN only matches NaN, an infinity the same infinity, probe
scores (one nonzero product) exact, finite scores of mixed corpora within oracle.scoring.TOL; int8 and 1-bit exact.

  * page_rows_device, bit for bit: every bf16 pattern, e4m3 code, int8 code and sign byte, at scale 1 and 0.3.
  * Probes: single-row sources holding one value in element i against one-hot pages (1, 2^64, -2^-64 and 2^-100 for bf16):
    every bf16 pattern and e4m3 code on the A operand, products that overflow, land in fp32's subnormal range or underflow.
    A product in fp32's subnormal range comes back rounded toward zero, as the value rule states.
  * Non-finite sources (+-inf, NaN, mixed signs across rows, +inf meeting -inf in a row) of 1 .. 65 rows against the value
    suite's non-finite pages; bit-identical to search_device of the same rows over the length.
  * The int8 bound through page sources (1023 / 1024 rows of -128, 1041 rows of +-127), MMR sims on them, an example fused
    after the clamp; 1-bit sources against an int64 (128 - hamming) oracle.
  * Examples whose scores are infinite or NaN, fused against a numpy float32 fusion; a page the mask forbids never appears.
  * zero_pad_compat does not apply to the page and example calls, on the index and through the store.
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

import float_value_oracle as fvo  # noqa: E402
import page_query_oracle as pqo  # noqa: E402
from explain_oracle import similarity_np  # noqa: E402
from morphik_core_b200 import _native as nat  # noqa: E402
from morphik_core_b200.index import MaxSimIndex  # noqa: E402
from morphik_core_b200.models import DocumentChunk  # noqa: E402
from morphik_core_b200.store import B200MultiVectorStore  # noqa: E402
from oracle import maxsim_oracle as orc  # noqa: E402
from oracle.scoring import TOL, i32_reported, i32_sum  # noqa: E402
from test_gpu_mmr import check_sims, run_mmr  # noqa: E402
from test_gpu_scorer_values import (J0, J1, J2, assert_values, candidate_lists, check_candidates,  # noqa: E402
                                    check_ranking, pad_pages, same_values, special_corpus)

DEV = torch.device("cuda", 0)
INF, NAN = np.inf, np.nan
UNIT = {"bf16": 1.0, "fp8": fvo.F8_SCALE ** 2}
EDGE_LENS = [1, 31, 32, 33, 64, 65]


_OPEN = []  # indexes and stores a test made, closed after it


def track(x):
    _OPEN.append(x)
    return x


@pytest.fixture(autouse=True)
def close_what_the_test_opened():
    yield
    torch.cuda.synchronize()
    while _OPEN:
        _OPEN.pop().close()


def host(ts):
    torch.cuda.synchronize()
    return tuple(t.cpu().numpy() for t in ts)


def bits(x):
    return np.ascontiguousarray(x, np.float32).view(np.uint32)


def packed_index(dtype, rows_u8, lens):
    idx = track(MaxSimIndex(dtype=dtype))
    idx.append_packed(torch.from_numpy(np.ascontiguousarray(pad_pages(rows_u8, lens))).to(DEV), [int(n) for n in lens])
    idx._attach()
    return idx


def stored_values(idx, dtype):
    """Every page's true rows as the packed values the scan multiplies (float64, fvo's units)."""
    raw = idx.packed_rows().cpu().numpy()
    start = pqo.starts_of(idx.page_lens)
    return [fvo.packed_values(dtype, raw[start[p]:start[p] + n]) for p, n in enumerate(idx.page_lens)]


def scattered(ts, ti, tc, n_pages, offset=0):
    """Per source, the reported score of every returned page at column id - offset (NaN-filled elsewhere is not used)."""
    out = np.full((len(tc), n_pages), np.nan, np.float32)
    for i in range(len(tc)):
        n = int(tc[i])
        out[i, ti[i, :n] - offset] = ts[i, :n]
    return out


def assert_nan_bits(ts):
    nan = np.isnan(ts)
    assert (bits(ts)[nan] == 0x7FFFFFFF).all(), "a NaN score is reported as 0x7fffffff"


# ------------------------------------------------------------------------------------------------ page_rows_device
def value_rows(dtype):
    """uint8 rows [n, row bytes] holding every input value of the dtype, and their float64 values [n, 128]."""
    if dtype == "bf16":
        pats = np.arange(65536, dtype=np.uint32).astype(np.uint16).reshape(512, 128)
        return pats.view(np.uint8).reshape(512, 256), fvo.bf16_values(pats)
    if dtype == "fp8":
        codes = np.arange(256, dtype=np.uint8).reshape(2, 128)
        return codes, fvo.e4m3_values(codes)
    if dtype == "int8":
        codes = np.arange(-128, 128, dtype=np.int16).astype(np.int8).reshape(2, 128)
        return codes.view(np.uint8), codes.astype(np.float64)
    byts = np.arange(256, dtype=np.uint8).reshape(16, 16)
    return byts, np.where(np.unpackbits(byts, axis=1) > 0, 1.0, -1.0)


def page_rows_raw(idx, src, scale):
    n = int(sum(int(idx.page_lens[p]) for p in src))
    out = torch.empty((max(n, 1), 128), dtype=torch.float32, device=DEV)
    idx.h.check(nat.lib.b200ms_page_rows_device(idx.h.ptr, nat.i64_array(src), len(src), ctypes.c_float(scale),
                                                ctypes.c_void_p(out.data_ptr()), idx._stream()), "b200ms_page_rows_device")
    torch.cuda.synchronize()
    return out[:n].cpu().numpy()


@pytest.mark.parametrize("dtype", ["bf16", "fp8", "int8", "binary"])
def test_page_rows_every_value_bit_for_bit(dtype):
    raw, vals = value_rows(dtype)
    reps = -(-sum(EDGE_LENS) // len(raw))
    raw, vals = np.tile(raw, (reps, 1)), np.tile(vals, (reps, 1))
    lens = EDGE_LENS + ([len(raw) - sum(EDGE_LENS)] if len(raw) > sum(EDGE_LENS) else [])
    idx = packed_index(dtype, raw, lens)
    first = np.concatenate([[0], np.cumsum(lens)])
    src = list(reversed(range(len(lens)))) + [0, 3]
    want_vals = np.concatenate([vals[first[p]:first[p + 1]] for p in src]).astype(np.float32)
    for scale in (1.0, 0.3):
        got = page_rows_raw(idx, src, scale)
        with np.errstate(over="ignore", invalid="ignore"):
            want = want_vals * np.float32(scale)
        nan = np.isnan(want)
        assert np.array_equal(np.isnan(got), nan), (dtype, scale)
        bad = np.argwhere((bits(got) != bits(want)) & ~nan)
        assert len(bad) == 0, (dtype, scale, len(bad), [(tuple(b), got[tuple(b)], want[tuple(b)]) for b in bad[:4]])


# ------------------------------------------------------------------------------------------------ query-side probes
BF16_MULTS = [1.0, 2.0 ** 64, -(2.0 ** -64), 2.0 ** -100]
F8_MULT_CODES = [0x38, 0xFE, 0x01]  # 1.0, -448, 2^-9


def probe_corpus(dtype):
    """(index, n_src, source values [n_src] at element s % 128, one-hot values [n_mult], their elements): single-row sources
    holding every value, then one-hot pages (value m at element j, for every multiplier and j)."""
    if dtype == "bf16":
        v_bits = np.arange(65536, dtype=np.uint32).astype(np.uint16)
        m_bits = (np.asarray(BF16_MULTS, np.float32).view(np.uint32) >> 16).astype(np.uint16)
        elem = np.uint16
        values, mvals = fvo.bf16_values(v_bits), fvo.bf16_values(m_bits)
    else:
        v_bits = np.arange(256, dtype=np.uint8)
        m_bits = np.asarray(F8_MULT_CODES, np.uint8)
        elem = np.uint8
        values, mvals = fvo.e4m3_values(v_bits), fvo.e4m3_values(m_bits)
    n_src = len(v_bits)
    src_rows = np.zeros((n_src, 128), elem)
    src_rows[np.arange(n_src), np.arange(n_src) % 128] = v_bits
    oh = np.zeros((len(m_bits) * 128, 128), elem)
    oh_j = np.tile(np.arange(128), len(m_bits))
    oh[np.arange(len(oh)), oh_j] = np.repeat(m_bits, 128)
    rows = np.concatenate([src_rows, oh]).view(np.uint8).reshape(n_src + len(oh), -1)
    idx = packed_index(dtype, rows, [1] * len(rows))
    return idx, n_src, values, np.repeat(mvals, 128), oh_j


def probe_expected(values, s_elem, ohv, oh_j):
    """[n, n_onehot]: v * m exactly rounded to fp32 where the elements meet, else 0 * v (NaN for a non-finite v)."""
    with np.errstate(over="ignore", invalid="ignore"):
        prod = fvo.fp32(values[:, None] * ohv[None, :])
    meet = s_elem[:, None] == oh_j[None, :]
    return np.where(meet, prod, np.where(np.isfinite(values)[:, None], 0.0, np.nan))


@pytest.mark.parametrize("dtype", ["bf16", "fp8"])
def test_every_value_on_the_query_operand(dtype):
    idx, n_src, values, ohv, oh_j = probe_corpus(dtype)
    n_oh = len(ohv)
    allow = np.zeros(idx.n_pages, bool)
    allow[n_src:] = True
    masks = torch.from_numpy(idx.mask_from_pages(allow)[None].view(np.int32)).to(DEV)
    unit = UNIT[dtype]
    cand = torch.arange(n_src, idx.n_pages, dtype=torch.int64, device=DEV).flip(0)
    for name, step in (("search_pages", 4096), ("rerank_pages_batch", 1024)):
        for s0 in range(0, n_src, step):
            src = list(range(s0, min(s0 + step, n_src)))
            index = torch.zeros(len(src), dtype=torch.int32, device=DEV)
            if name == "search_pages":
                ts, ti, tc = host(idx.search_pages(src, n_oh, masks, index))
            else:
                ts, ti, tc = host(idx.rerank_pages_batch(src, cand.repeat(len(src), 1).contiguous(), n_oh))
            assert (tc == n_oh).all(), name
            assert_nan_bits(ts)
            got = scattered(ts, ti, tc, n_oh, n_src).astype(np.float64) * unit
            want = probe_expected(values[src], np.asarray(src) % 128, ohv, oh_j)
            assert_values(got, want, 0.0, f"{dtype} {name} sources {s0}..")
            for i in range(0, len(src), 97):  # the order: NaN first, then +inf, finite DESC, -inf; ties by id (slot)
                if name == "search_pages":
                    assert np.array_equal(ti[i], orc.topk_np(want[i], n_oh)[1] + n_src), (name, src[i])
                else:  # slot j holds page n_pages - 1 - j
                    slots = orc.topk_np(want[i][::-1].copy(), n_oh)[1]
                    assert np.array_equal(ti[i], idx.n_pages - 1 - slots), (name, src[i])
    if dtype == "bf16":  # the products the multipliers make: overflow, subnormal results and underflow to 0 all occur
        want = probe_expected(values, np.arange(n_src) % 128, ohv, oh_j)
        fin = np.isfinite(values)[:, None] & (np.arange(n_src) % 128 == 0)[:, None]
        assert (np.isinf(want) & fin).any() and ((np.abs(want) < 2.0 ** -126) & (want != 0) & fin).any()
        assert ((want == 0) & fin & (values != 0)[:, None] & (oh_j == 0)[None, :]).any()
        with np.errstate(over="ignore", invalid="ignore"):  # and products whose subnormal result truncation changes
            x = values[np.isfinite(values)][:, None] * np.asarray(BF16_MULTS)[None, :]
            assert (fvo.fp32(x) != x.astype(np.float32)).any()


# ------------------------------------------------------------------------------------------------ non-finite sources
SRC_KINDS = ["inf", "neginf", "nan", "inf_mixed_rows", "inf_cancel_in_row"]


@functools.lru_cache(maxsize=None)
def nonfinite_pages():
    """(pages float32, index of the first source): the value suite's non-finite pages, then a source of every kind and
    length."""
    pages, _ = special_corpus()
    pages = list(pages)
    first = len(pages)
    rng = np.random.default_rng(88)
    for kind in SRC_KINDS:
        for n in EDGE_LENS:
            d = (rng.standard_normal((n, 128)) / np.sqrt(128)).astype(np.float32)
            d[:, [J0, J1, J2]] = 0.25 * np.where(np.arange(n) % 3 == 0, -1, 1)[:, None]
            if kind == "inf":
                d[:, J0] = INF
            elif kind == "neginf":
                d[:, J0] = -INF
            elif kind == "nan":
                d[n // 2, J1] = NAN
            elif kind == "inf_mixed_rows":
                d[:, J0] = np.where(np.arange(n) % 2, INF, -INF)
            else:
                d[:, J0], d[:, J2] = INF, -INF
            pages.append(d)
    return pages, first


@pytest.fixture(scope="module")
def nonfinite():
    """dtype -> (index, sources, want [n_src, n_pages], slack [n_src, n_pages]): want is the oracle's reported score over
    the source's length; slack bounds the rounding of a finite score by the magnitude of its terms, 4 * TOL * (sum over
    tokens of the largest sum of |products| of a row), so that sums that cancel large terms are held to what fp32 can
    keep of them."""
    made = {}

    def get(dtype):
        if dtype not in made:
            pages, first = nonfinite_pages()
            idx = MaxSimIndex(dtype=dtype)
            idx.add_pages(pages)
            idx._attach()
            vals = stored_values(idx, dtype)
            src = [2] + list(range(first, len(pages)))  # page 2: a finite page of the value suite's corpus
            lens = np.asarray([len(vals[p]) for p in src], np.float32)[:, None]
            reported = fvo.fp32(fvo.scores([vals[p] for p in src], vals) / UNIT[dtype]).astype(np.float32)
            want = (reported / lens).astype(np.float64)  # over the length in fp32, as __fdiv_rn
            fin = [np.abs(np.where(np.isfinite(v), v, 0.0)) for v in vals]
            mag = fvo.scores([fin[p] for p in src], fin) / UNIT[dtype] / lens
            made[dtype] = (idx, src, want, 4 * TOL[dtype] * np.maximum(mag, 1e-3))
        return made[dtype]

    yield get
    torch.cuda.synchronize()
    for idx, *_ in made.values():
        idx.close()


def check_order_with_slack(ts, ti, tc, ws, wi, want, slack, what):
    """A top-k against the oracle's order (ws, wi): non-finite positions exactly the oracle's id and class; a finite
    position within slack of the oracle, and holding another id only where the two ids' oracle scores tie within slack."""
    n = len(wi)
    assert int(tc) == n and (ti[n:] == -1).all(), (what, int(tc), n)
    for j in range(n):
        p, q = int(ti[j]), int(wi[j])
        if not np.isfinite(ws[j]):
            assert p == q and len(same_values([ts[j]], [ws[j]])) == 0, (what, j, p, q, ts[j], ws[j])
            continue
        assert np.isfinite(want[p]) and abs(float(ts[j]) - want[p]) <= slack[p], (what, j, p, ts[j], want[p], slack[p])
        assert p == q or abs(want[p] - ws[j]) <= slack[p] + slack[q], (what, j, p, q, want[p], ws[j])


@pytest.mark.parametrize("dtype", ["bf16", "fp8"])
def test_non_finite_sources(dtype, nonfinite):
    idx, src, want, slack = nonfinite(dtype)
    n = idx.n_pages
    assert np.isnan(want).any() and np.isfinite(want).any()
    if dtype == "bf16":
        assert (want == INF).any() and (want == -INF).any()
    ts, ti, tc = host(idx.search_pages(src, n))
    assert_nan_bits(ts)
    first = nonfinite_pages()[1]
    # fp8 saturates the infinities to +-448: where +448 and -448 rows meet, a finite sum cancels products of 448 * 16, and
    # the fp32 rounding of those terms is far beyond TOL of the small result, so those sources get the magnitude slack
    cancel = [first + SRC_KINDS.index(k) * len(EDGE_LENS) + j for k in ("inf_mixed_rows", "inf_cancel_in_row")
              for j in range(len(EDGE_LENS))] if dtype == "fp8" else []
    for i, p in enumerate(src):
        what = f"{dtype} search_pages source {p}"
        if p in cancel:
            ws, wi = orc.topk_np(want[i], n)
            check_order_with_slack(ts[i], ti[i], tc[i], ws, wi, want[i], slack[i], what)
        else:
            check_ranking(dtype, ts[i], ti[i], tc[i], want[i], n, what=what)
    cand = candidate_lists(n, len(src), 31)
    ts, ti, tc = host(idx.rerank_pages_batch(src, torch.from_numpy(cand).to(DEV), n))
    for i, p in enumerate(src):
        what = f"{dtype} rerank_pages_batch source {p}"
        if p in cancel:
            ws, wi = slot_order(want[i], cand[i], np.ones(n, bool), n)
            check_order_with_slack(ts[i], ti[i], tc[i], ws, wi, want[i], slack[i], what)
        else:
            check_candidates(dtype, ts[i], ti[i], tc[i], want[i], cand[i], n, what)
    # bit for bit search_device's scores of the same rows over the length: NaN, +-inf and -0 / +0 included
    rows, lens = idx.page_rows(src)
    ws, wi, wc = host(idx.search_device(rows[:sum(lens)].contiguous(), lens, n))
    ws = ws / np.asarray(lens, np.float32)[:, None]
    ts, ti, tc = host(idx.search_pages(src, n))
    assert np.array_equal(tc, wc) and np.array_equal(ti, wi)
    nan = np.isnan(ws)
    assert np.array_equal(np.isnan(ts), nan) and np.array_equal(bits(ts)[~nan], bits(ws)[~nan])


def slot_order(want, cand, allow, k):
    """The oracle's order of a candidate list: (scores, page ids) of its valid slots that `allow` keeps, ties by slot."""
    valid = (cand >= 0) & (cand < len(want))
    valid[valid] &= allow[cand[valid]]
    ws, slots = orc.topk_np(np.where(valid, want[np.where(valid, cand, 0)], 0.0), k, valid)
    return ws, cand[slots]


# ------------------------------------------------------------------------------------------------ int8 bound
def i8_bound_pages():
    alt = np.where(np.arange(128) % 2, 127, -127).astype(np.int8)
    plus = np.full(128, 127, np.int8)
    pm = np.stack([plus if r % 2 == 0 else alt for r in range(1041)])
    rng = np.random.default_rng(6)
    return [np.full((1023, 128), -128, np.int8),    # 0: 1023 * 2^21 = 2^31 - 2^21 against page 2
            np.full((1024, 128), -128, np.int8),    # 1: 1024 * 2^21 = 2^31, clamped
            np.full((1, 128), -128, np.int8),       # 2
            pm,                                     # 3: 1041 rows of +-127 against page 4: past the bound
            np.stack([plus, alt]),                  # 4
            rng.integers(-128, 128, (40, 128)).astype(np.int8),
            np.full((1, 128), -128, np.int8),       # 6: a copy of page 2 (a tie at the bound: lower id first)
            np.zeros((0, 128), np.int8)]


def test_int8_bound_through_page_sources():
    pages = i8_bound_pages()
    lens = [len(p) for p in pages]
    idx = packed_index("int8", np.concatenate([p for p in pages if len(p)]).view(np.uint8), lens)
    n, s = idx.n_pages, idx.score_scale
    sums = np.array([[similarity_np(pages[a], pages[b], "int8").max(axis=1).sum() if lens[a] and lens[b] else 0
                      for b in range(n)] for a in range(n)], np.int64)
    assert sums[0, 2] == 2 ** 31 - 2 ** 21 and sums[1, 2] == 2 ** 31 and sums[3, 4] > 2 ** 31 > 1040 * 127 * 127 * 128
    src = [0, 1, 3, 5]

    def reported(a):
        return i32_reported(sums[a], s) / np.float32(lens[a])

    ts, ti, tc = host(idx.search_pages(src, n))
    for i, a in enumerate(src):
        ws, wi = orc.topk_np(i32_sum(sums[a]).astype(np.float64), n)
        assert int(tc[i]) == len(wi) and np.array_equal(ti[i, :len(wi)], wi), a
        assert np.array_equal(bits(ts[i, :len(wi)]), bits(reported(a)[wi])), a
    assert list(ti[1, :4]) == [0, 1, 2, 6] and len(set(bits(ts[1, :4]).tolist())) == 1  # clamped, tied, lower id first
    cand = np.stack([np.random.default_rng(a).permutation(n) for a in src]).astype(np.int64)
    cand[:, 3] = -1
    ts, ti, tc = host(idx.rerank_pages_batch(src, torch.from_numpy(cand).to(DEV), n))
    for i, a in enumerate(src):
        valid = cand[i] >= 0
        keys = np.where(valid, i32_sum(sums[a])[np.maximum(cand[i], 0)], 0).astype(np.float64)
        _, slots = orc.topk_np(keys, n, valid)
        assert int(tc[i]) == len(slots) and np.array_equal(ti[i, :len(slots)], cand[i][slots]), a
        assert np.array_equal(bits(ts[i, :len(slots)]), bits(reported(a)[cand[i][slots]])), a
    # MMR sims between these pages: exact int64 sums, no clamp
    ids = np.array([[0, 1, 2, 3, 4, 6]], np.int64)
    got = run_mmr(idx, ids, np.array([[6, 5, 4, 3, 2, 1]], np.float32), [1], 6, 0.5)
    check_sims("int8", ids, got, pages, s)
    # an example fuses the clamped value
    w = [0.5, -0.25]
    ts, ti, tc = host(idx.search_examples(None, [], [1, 0], [0, 0], w, 1, n))
    fused = pqo.fuse(np.stack([reported(1), reported(0)]), w)
    _, wi = orc.topk_np(fused.astype(np.float64), n)
    assert int(tc[0]) == n and np.array_equal(ti[0], wi)
    assert np.array_equal(bits(ts[0]), bits(fused[wi]))


# ------------------------------------------------------------------------------------------------ 1-bit sources
def test_binary_sources_against_hamming():
    rng = np.random.default_rng(12)
    lens = [1, 31, 32, 33, 64, 65, 100, 0, 5, 2]
    raw = rng.integers(0, 256, (sum(lens), 16)).astype(np.uint8)
    raw[35] = raw[0]  # a row shared by two pages
    idx = packed_index("binary", raw, lens)
    first = np.concatenate([[0], np.cumsum(lens)])
    pages = [raw[first[p]:first[p + 1]] for p in range(len(lens))]
    n = len(lens)
    S = np.array([[similarity_np(pages[a], pages[b], "bits").max(axis=1).sum() if lens[a] and lens[b] else 0
                   for b in range(n)] for a in range(n)], np.int64)
    src = [0, 1, 2, 3, 4, 5, 6, 8, 9, 4]
    ts, ti, tc = host(idx.search_pages(src, n))
    cand = np.stack([np.random.default_rng(a).permutation(n) for a in range(len(src))]).astype(np.int64)
    cand[:, 5] = -1
    rs, ri, rc = host(idx.rerank_pages_batch(src, torch.from_numpy(cand).to(DEV), n))
    for i, a in enumerate(src):
        rep = i32_reported(S[a], idx.score_scale) / np.float32(lens[a])
        ws, wi = orc.topk_np(S[a].astype(np.float64), n)
        assert int(tc[i]) == n and np.array_equal(ti[i], wi) and np.array_equal(bits(ts[i]), bits(rep[wi])), a
        valid = cand[i] >= 0
        _, slots = orc.topk_np(np.where(valid, S[a][np.maximum(cand[i], 0)], 0).astype(np.float64), n, valid)
        assert int(rc[i]) == len(slots) and np.array_equal(ri[i, :len(slots)], cand[i][slots]), a
        assert np.array_equal(bits(rs[i, :len(slots)]), bits(rep[cand[i][slots]])), a


# ------------------------------------------------------------------------------------------------ non-finite examples
def test_examples_with_non_finite_scores(nonfinite):
    idx, src, want, _ = nonfinite("bf16")
    n = idx.n_pages
    first = nonfinite_pages()[1]
    row = {(k, ln): first + SRC_KINDS.index(k) * len(EDGE_LENS) + EDGE_LENS.index(ln) for k in SRC_KINDS for ln in EDGE_LENS}
    per = {p: want[i] for i, p in enumerate(src)}
    requests = [  # (page examples, weights); page 2 is a finite page of the value suite's corpus
        ([row["inf", 33], row["nan", 31]], [1.0, 0.5]),         # a NaN example
        ([row["inf", 31], row["inf", 64]], [1.0, -1.5]),        # +inf meets -inf across examples
        ([2, row["inf", 1], row["neginf", 65]], [1.0, -0.25, 0.5]),  # a negative weight times +inf
    ]
    ex, req, w = [], [], []
    for r, (pages, ws) in enumerate(requests):
        ex += pages
        req += [r] * len(pages)
        w += ws
    fused = np.stack([pqo.fuse(np.stack([per[p] for p in pages]), ws) for pages, ws in requests]).astype(np.float64)
    mag = np.stack([sum(abs(x) * np.abs(np.nan_to_num(per[p], nan=0, posinf=0, neginf=0)) for p, x in zip(pages, ws))
                    for pages, ws in requests])
    assert np.isnan(fused[1]).sum() > np.isnan(np.stack([per[p] for p in requests[1][0]])).any(axis=0).sum()
    assert np.isneginf(fused[2]).any() and np.isnan(fused[0]).any()
    # requests 1 and 2 may not return their NaN pages
    allow = np.ones((3, n), bool)
    allow[1:] = ~np.isnan(fused[1:])
    assert (~allow[1]).any()
    masks = torch.from_numpy(np.stack([idx.mask_from_pages(a) for a in allow]).view(np.int32)).to(DEV)
    index = torch.tensor([-1, 1, 2], dtype=torch.int32, device=DEV)
    cand = candidate_lists(n, 3, 44)
    for name in ("search_examples", "rerank_examples_batch"):
        if name == "search_examples":
            ts, ti, tc = host(idx.search_examples(None, [], ex, req, w, 3, n, masks, index))
        else:
            ts, ti, tc = host(idx.rerank_examples_batch(None, [], ex, req, w, 3, torch.from_numpy(cand).to(DEV), n, masks,
                                                        index))
        for r in range(3):
            if name == "search_examples":
                ws, wi = orc.topk_np(fused[r], n, allow[r])
            else:
                ws, wi = slot_order(fused[r], cand[r], allow[r], n)
            assert allow[r][ti[r, :tc[r]]].all(), (name, r)
            check_order_with_slack(ts[r], ti[r], tc[r], ws, wi, fused[r], 4 * TOL["bf16"] * mag[r] + 1e-30,
                                   f"{name} request {r}")
            assert np.isnan(ts[r, :int(np.isnan(ws).sum())]).all()  # NaN ranks first


# ------------------------------------------------------------------------------------------------ zero_pad_compat
@functools.lru_cache(maxsize=None)
def zero_pad_pages():
    """Ragged pages, even ones all positive, odd ones all negative: a source of one sign against a page of the other has
    negative token maxima, which the clamp of a short page would raise to 0."""
    rng = np.random.default_rng(41)
    lens = [int(x) for x in rng.integers(1, 120, size=60)] + [0, 300, 2]
    return [(np.abs(rng.standard_normal((n, 128))) / np.sqrt(128) * (-1.0 if i % 2 else 1.0)).astype(np.float32)
            for i, n in enumerate(lens)]


@pytest.mark.parametrize("tier", ["hbm", "host"])
@pytest.mark.parametrize("dtype", ["bf16", "int8", "fp8"])
def test_zero_pad_compat_does_not_apply_to_page_and_example_calls(dtype, tier):
    """The four page and example calls give the same bits under the option as without it, on both tiers (the host tier's
    candidate rounds included; its full scans are refused).  Controls: search_device (a full scan, HBM) and rerank_batch
    (a candidate list, both tiers) of the same query rows change under the option, so the corpus exercises the clamp."""
    pages = zero_pad_pages()
    n = len(pages)
    idx = track(MaxSimIndex(dtype=dtype, tier=tier))
    idx.add_pages(pages)
    src = [1, 2, 5, 61, 8]
    rng = np.random.default_rng(3)
    cand = torch.from_numpy(np.stack([rng.permutation(n)[:40] for _ in range(len(src))]).astype(np.int64)).to(DEV)
    qlens = [len(pages[3]), len(pages[4])]  # one negative and one positive page's rows as query examples
    q = torch.from_numpy(np.concatenate([pages[3], pages[4]])).to(DEV)
    ex_pages, ex_req, ex_w = [1, 2, 61], [0, 0, 1, 1, 0], [1.0, -0.5, 1.0, 0.5, 0.25]  # query examples first
    calls = {
        "rerank_pages_batch": lambda: idx.rerank_pages_batch(src, cand, 40),
        "rerank_examples_batch": lambda: idx.rerank_examples_batch(q, qlens, ex_pages, ex_req, ex_w, 2,
                                                                   cand[:2].contiguous(), 40),
        "rerank_batch": lambda: idx.rerank_batch(q, qlens, cand[:2].contiguous(), 40),
    }
    if tier == "hbm":
        calls.update({
            "search_pages": lambda: idx.search_pages(src, n),
            "search_examples": lambda: idx.search_examples(q, qlens, ex_pages, ex_req, ex_w, 2, n),
            "search_device": lambda: idx.search_device(q, qlens, n),
        })
    controls = ("search_device", "rerank_batch")

    def run():
        return {name: host(f()) for name, f in calls.items()}

    base = run()
    for batch in (1, 3, 128):
        idx.set_option("zero_pad_compat", batch)
        got = run()
        for name, out in got.items():
            same = all(np.array_equal(a.view(np.uint8), b.view(np.uint8)) for a, b in zip(out, base[name]))
            if name in controls:  # the clamp changes these wherever a batch has pages of different lengths
                assert same == (batch == 1), (dtype, tier, batch, name)
            else:
                assert same, (dtype, tier, batch, name)
    idx.set_option("zero_pad_compat", 0)


def test_store_similar_and_feedback_ignore_zero_pad_compat():
    pages = zero_pad_pages()
    stores = []
    for zp in (0, 128):
        store = track(B200MultiVectorStore(mode="bf16", coalesce_queries=False, zero_pad_compat=zp))
        chunks = [DocumentChunk(document_id=f"d{i // 4}", chunk_number=i % 4, content="", embedding=p, metadata={})
                  for i, p in enumerate(pages) if len(p)]
        asyncio.run(store.store_embeddings(chunks))
        stores.append(store)

    def key(res):
        return [(c.document_id, c.chunk_number, np.float32(c.score).view(np.uint32).item()) for c in res]

    out = []
    for store in stores:
        sim = asyncio.run(store.query_similar_to_chunks([("d0", 1), ("d3", 2), ("d10", 0)], k=30,
                                                        include_same_document=True))
        fb = asyncio.run(store.query_similar_with_feedback(-np.abs(pages[4]), k=30, positive_chunks=[("d0", 1)],
                                                           negative_chunks=[("d2", 2)]))
        out.append(([key(r) for r in sim], key(fb)))
    assert out[0] == out[1]
    assert all(len(r) for r in out[0][0]) and len(out[0][1])
