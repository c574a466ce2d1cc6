"""The plan rule of a filtered full scan (tests/scan_plan_model.py), on random and hand-made inputs; no GPU.
tests/test_gpu_filtered_scan.py holds the kernels of csrc/scan_plan.cu to this model."""
import numpy as np
import pytest

import scan_plan_model as spm

SMS = 132


def ragged_lens(rng, n):
    lens = rng.integers(1, 1031, size=n)
    lens[rng.random(n) < 0.1] = 0
    lens[:9] = [0, 1, 31, 32, 33, 0, 0, 1030, 1024]
    return [int(x) for x in lens]


def check_plan(p, allow, lens, cap, num_sms=SMS):
    pad = spm.padded(lens)
    start = np.concatenate([[0], np.cumsum(pad)]) // spm.CHUNK
    chunk_page = np.repeat(np.arange(len(pad)), pad // spm.CHUNK)
    covered = []
    last_end = 0
    ur = spm.unit_rows_for(int(pad[allow].sum()), num_sms, cap)
    for c0, c1 in p.units:
        assert last_end <= c0 < c1  # ascending, disjoint, not empty
        last_end = c1
        pages = np.unique(chunk_page[c0:c1])
        assert c0 == start[pages[0]] and c1 == start[pages[-1] + 1]  # whole pages
        assert allow[pages].all()  # no page with rows in the unit is disallowed
        assert (c1 - c0) * spm.CHUNK < ur + pad[pages[-1]]  # below the cap plus its last page
        covered.extend(pages.tolist())
    want = [int(x) for x in np.flatnonzero(allow & (pad > 0))]
    assert covered == want  # exactly the allowed pages that have rows, each once
    assert p.pages == [int(x) for x in np.flatnonzero(allow)]
    assert p.rows == int(pad[allow].sum()) == sum((c1 - c0) * spm.CHUNK for c0, c1 in p.units)


@pytest.mark.parametrize("seed", range(6))
@pytest.mark.parametrize("frac", [0.0, 0.001, 0.01, 0.1, 0.5, 0.99, 1.0])
def test_random_masks_give_whole_page_units_over_exactly_the_allowed_pages(seed, frac):
    rng = np.random.default_rng(100 * seed + int(frac * 1000))
    lens = ragged_lens(rng, int(rng.integers(40, 4000)))
    allow = rng.random(len(lens)) < frac
    cap = int(rng.choice([128, 400, 4096]))
    check_plan(spm.plan(spm.mask_words(allow), None, lens, SMS, cap), allow, lens, cap)


def test_all_ones_is_the_corpus_plan_and_all_zeros_is_empty():
    rng = np.random.default_rng(5)
    for n, cap in ((3000, 4096), (777, 128), (50, 4096), (20000, 1024)):
        lens = ragged_lens(rng, n)
        full = [(c0, c1) for c0, c1, _, _ in spm.corpus_units(lens, SMS, cap)]
        ones = spm.plan(spm.mask_words(np.ones(n, bool)), None, lens, SMS, cap)
        assert ones.units == full and ones.rows == int(spm.padded(lens).sum())
        zeros = spm.plan(spm.mask_words(np.zeros(n, bool)), None, lens, SMS, cap)
        assert zeros.units == [] and zeros.pages == [] and zeros.rows == 0


def test_bits_past_the_last_page_are_ignored():
    rng = np.random.default_rng(6)
    lens = ragged_lens(rng, 1001)  # 1001 % 32 != 0: the last word has 23 spare bits
    allow = rng.random(1001) < 0.3
    a = spm.plan(spm.mask_words(allow), None, lens, SMS)
    b = spm.plan(spm.mask_words(allow, set_tail=True), None, lens, SMS)
    assert (a.units, a.pages, a.rows) == (b.units, b.pages, b.rows)


def test_mask_index_names_the_union_and_minus_one_means_every_page():
    rng = np.random.default_rng(7)
    lens = ragged_lens(rng, 2500)
    n = len(lens)
    rows = [rng.random(n) < f for f in (0.02, 0.2, 0.5)]
    masks = np.stack([spm.mask_words(r) for r in rows])
    p = spm.plan(masks, [0, 1, 1, 0], lens, SMS)
    check_plan(p, rows[0] | rows[1], lens, 4096)  # row 2 is named by no query
    assert p.units == spm.plan(spm.mask_words(rows[0] | rows[1]), None, lens, SMS).units
    full = spm.plan(masks, [0, -1, 2], lens, SMS)
    assert full.units == [(c0, c1) for c0, c1, _, _ in spm.corpus_units(lens, SMS, 4096)]
    assert full.pages == list(range(n))


def test_hand_made_corpus():
    # 10 pages of 128 rows; unit_rows clamps to 128, so the corpus' plan is one unit per page
    lens = [128] * 10
    allow = np.array([1, 1, 0, 1, 0, 0, 1, 1, 1, 0], bool)
    p = spm.plan(spm.mask_words(allow), None, lens, SMS)
    assert p.units == [(0, 4), (4, 8), (12, 16), (24, 28), (28, 32), (32, 36)] and p.rows == 6 * 128
    # one SM and a cap of 4096: the corpus' plan is units of three pages (rows / 4 = 320, reached by the third page), and the
    # filtered units are runs inside them, cut at 6 * 128 / 4 = 192 rows
    p = spm.plan(spm.mask_words(allow), None, lens, 1)
    assert spm.corpus_units(lens, 1, 4096) == [(0, 12, 0, 3), (12, 24, 3, 6), (24, 36, 6, 9), (36, 40, 9, 10)]
    assert p.units == [(0, 8), (12, 16), (24, 32), (32, 36)]
    # empty pages between allowed pages break nothing, disallowed or not
    lens = [256, 0, 0, 256, 256, 0, 256]
    p = spm.plan(spm.mask_words(np.array([1, 0, 1, 1, 0, 1, 1], bool)), None, lens, 1)
    assert spm.unit_rows_for(768, 1, 4096) == 192
    assert p.units == [(0, 8), (8, 16), (24, 32)] and p.pages == [0, 2, 3, 5, 6]
