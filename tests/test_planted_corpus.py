"""CPU checks of the test infrastructure the GPU path matrix stands on (no GPU needed):

* the int8 oracle's zero_pad_compat switch (C against numpy, both against the float oracle on integer-valued inputs);
* oracle.scoring.oracle_scores against the dtype-specific oracle calls it wraps;
* the planted-maximum corpora: every designated row is observable -- deleting it, moving a page boundary by a row or a chunk,
  or dropping a page's last chunk moves some page's oracle score by more than 10x the dtype's tolerance.  Without the
  plants (the control) some of those mutations go unseen, which is why random corpora cannot catch them.
"""
import numpy as np
import pytest

from oracle import maxsim_oracle as orc
from oracle import planted
from oracle.scoring import TOL, assert_scores, oracle_scores, score_error

DTYPES = ["bf16", "fp8", "int8", "binary"]


# ------------------------------------------------------------------------------------------------ int8 zero-pad oracle
@pytest.mark.parametrize("batch", [1, 3, 7, 128])
def test_int8_zero_pad_oracle_c_matches_numpy_and_float_oracle(batch):
    rng = np.random.default_rng(40 + batch)
    lens = [0, 1, 5, 17, 3, 3, 40, 0, 2, 33, 9, 1, 64, 12, 8, 8, 0, 25]
    off = orc.page_offsets(lens)
    rows = rng.integers(-8, 9, size=(int(off[-1]), 128)).astype(np.int8)
    rows[off[2]:off[3]] = np.abs(rows[off[2]:off[3]])  # non-negative page: a negative query token has a negative maximum
    for q in (rng.integers(-8, 9, size=(7, 128)), -np.abs(rng.integers(1, 9, size=(5, 128))), rng.integers(-8, 9, size=(1, 128))):
        q = q.astype(np.int8)
        clean_c = orc.int8_maxsim_c(q, rows, off)
        assert np.array_equal(clean_c, orc.int8_maxsim_np(q, rows, off))
        zc = orc.int8_maxsim_c(q, rows, off, zero_pad_compat=True, batch=batch)
        zn = orc.int8_maxsim_np(q, rows, off, zero_pad_compat=True, batch=batch)
        assert np.array_equal(zc, zn)
        # integer-valued float inputs: the float oracle's switch gives the same numbers (sums stay below 2^24: exact)
        zf = orc.float_maxsim_c(q.astype(np.float32), rows.astype(np.float32), off, zero_pad_compat=True, batch=batch)
        assert np.array_equal(zc, zf.astype(np.int64))
        cf = orc.float_maxsim_c(q.astype(np.float32), rows.astype(np.float32), off)
        assert np.array_equal(clean_c, cf.astype(np.int64))
        # the clamp only ever raises a score, never on the longest page of a batch, and empty pages stay 0 unless padded
        assert np.all(zc >= clean_c)
        for p, n in enumerate(lens):
            b0 = p // batch * batch
            if n == max(lens[b0:b0 + batch]):
                assert zc[p] == clean_c[p]
    # the all-negative query really exercises the clamp
    qn = -np.abs(rng.integers(1, 9, size=(4, 128))).astype(np.int8)
    assert not np.array_equal(orc.int8_maxsim_c(qn, rows, off, True, 3), orc.int8_maxsim_c(qn, rows, off))


def test_oracle_scores_wraps_the_dtype_oracles():
    rng = np.random.default_rng(3)
    lens = [5, 0, 40, 33, 1]
    pages = [rng.standard_normal((n, 128)).astype(np.float32) * 0.1 for n in lens]
    qs = [rng.standard_normal((t, 128)).astype(np.float32) * 0.1 for t in (3, 32)]
    rows, off = np.concatenate(pages), orc.page_offsets(lens)
    for zp in (0, 2):
        w = oracle_scores("int8", qs, pages, zp)
        want = np.stack([orc.int8_maxsim_np(orc.quantize_int8_np(q, 127.0), orc.quantize_int8_np(rows, 127.0), off, zp > 0,
                                            zp or 128) for q in qs]) / 127.0 ** 2
        assert np.array_equal(w, want)
        w = oracle_scores("bf16", qs, pages, zp)
        want = np.stack([orc.float_maxsim_np(orc.bf16_round_np(q), orc.bf16_round_np(rows), off, zp > 0, zp or 128) for q in qs])
        assert_scores("bf16", w, want)
    b = oracle_scores("binary", qs, pages)
    assert np.array_equal(b[1], orc.binary_maxsim_np(orc.sign_pack_np(qs[1]), orc.sign_pack_np(rows), off)[0])
    f = oracle_scores("fp8", qs, pages)
    deq = lambda a: orc.dequantize_e4m3_np(orc.quantize_e4m3_np(a, 64.0)).astype(np.float64)  # noqa: E731
    assert_scores("fp8", f[0], orc.float_maxsim_np(deq(qs[0]), deq(rows), off) / 4096.0)
    with pytest.raises(ValueError):
        oracle_scores("binary", qs, pages, 3)


# ------------------------------------------------------------------------------------------------ planted corpora
def _moved(dtype, new, old):
    """True when a score moved by more than 10x the dtype's tolerance (exact dtypes: by at least one quantum)."""
    return score_error(dtype, np.atleast_1d(new), np.atleast_1d(old)) > (10 * TOL[dtype] if TOL[dtype] else 0.5)


def _mutations(pc):
    """(description, first page, mutated pages) for every mutation of every page / boundary."""
    pages = pc.pages
    for p, marks in pc.designated.items():
        for r, d in marks:
            yield f"delete row {r} (direction {d}) of page {p}", p, [np.delete(pages[p], r, axis=0)]
        n = len(pages[p])
        if n:
            cut = (n - 1) // 32 * 32
            yield f"drop the last chunk of page {p}", p, [pages[p][:cut]]
        if p + 1 < len(pages) and n and len(pages[p + 1]):
            a, b = pages[p], pages[p + 1]
            for s in (1, 32):
                if len(a) > s:
                    yield f"move {s} rows of page {p} to page {p + 1}", p, [a[:-s], np.concatenate([a[-s:], b])]
                if len(b) > s:
                    yield f"move {s} rows of page {p + 1} to page {p}", p, [np.concatenate([a, b[:s]]), b[s:]]


def _sensitivity(pc):
    q = [pc.directions.copy()]
    base = oracle_scores(pc.dtype, q, pc.pages)[0]
    unseen = []
    for what, p, new_pages in _mutations(pc):
        new = oracle_scores(pc.dtype, q, new_pages)[0]
        if not _moved(pc.dtype, new, base[p:p + len(new_pages)]):
            unseen.append(what)
    return unseen


@pytest.mark.parametrize("dtype", DTYPES)
def test_planted_corpus_makes_every_mutation_visible(dtype):
    pc = planted.planted_corpus(dtype, seed=11, n_random=6)
    lens = pc.lens
    assert min(n for n in lens if n) >= planted.D and 0 in lens
    starts = np.concatenate([[0], np.cumsum([(n + 31) // 32 * 32 for n in lens])])[:-1]
    assert {int(s) % 128 for s, n in zip(starts, lens) if n} == {0, 32, 64, 96}  # pages start in every tile column
    chunks = [(n + 31) // 32 for n in lens if n]
    assert any(c % 4 == 1 and c > 1 for c in chunks) and any(n % 32 for n in lens) and max(lens) > 400
    # designated rows sit on the boundary classes
    cols = {(r, int(s) + r) for p, s in enumerate(starts) for r, _ in pc.designated[p]}
    assert {g % 32 for _, g in cols} >= {0, 31} and {g % 128 for _, g in cols} >= {0, 127}
    planted.check_margins(pc)
    unseen = _sensitivity(pc)
    assert not unseen, unseen[:10]


@pytest.mark.parametrize("dtype", DTYPES)
def test_without_plants_mutations_go_unseen(dtype):
    """Control: the same corpus layout with the plants removed -- some row deletions no longer change any score."""
    pc = planted.planted_corpus(dtype, seed=11, n_random=6, strength_scale=0.0)
    assert _sensitivity(pc)


@pytest.mark.parametrize("dtype", DTYPES)
def test_planted_queries_score_the_designated_rows(dtype):
    """A query's score on every page is the sum of its tokens' planted maxima (the designated rows), within tolerance."""
    pc = planted.planted_corpus(dtype, seed=5, n_random=4)
    qs = planted.planted_queries(pc, [1, 33, 130], seed=2)
    got = oracle_scores(dtype, qs, pc.pages)
    for qi, q in enumerate(qs):
        for p, marks in pc.designated.items():
            if not marks:
                assert got[qi, p] == 0.0
                continue
            rows = np.stack([pc.pages[p][r] for r, _ in marks])
            want = oracle_scores(dtype, [q], [rows])[0, 0]  # the designated rows alone give the same score
            assert_scores(dtype, np.array([got[qi, p]]), np.array([want]), f"page {p}")
