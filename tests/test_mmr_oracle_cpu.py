"""The MMR oracle (tests/mmr_oracle.py) on hand-worked cases: the pick rule's order, ties, NaN, duplicate and unused slots,
empty pages, and page_sims against a brute-force scalar loop for every corpus kind."""
import numpy as np
import pytest

from explain_oracle import quantise
from mmr_oracle import greedy, order_key, page_sims, page_sum, relevance, sim_value, valid_slots

INF, NAN = np.inf, np.nan


def f32(*v):
    return np.asarray(v, np.float32)


def test_lambda_one_is_rel_order_and_never_reads_red():
    rel = f32(0.5, 0.9, 0.7, 0.9)
    sims = np.full((4, 4), INF, np.float32)  # 0 * inf would be NaN, which ranks first, if red were read
    assert greedy(rel, sims, 4, 1.0) == [1, 3, 2, 0]


def test_lambda_zero_takes_the_most_novel_page_after_the_first():
    rel = f32(1.0, 0.9, 0.1, 0.5)
    sims = np.zeros((4, 4), np.float32)
    sims[:, 0] = [0, 0.8, 0.3, 0.6]  # coverage by page 0
    sims[:, 2] = [0.1, 0.2, 0, 0.9]
    # pick 1 = slot 0 (best rel); then v = -red: slot 2 (0.3) beats 3 (0.6) and 1 (0.8); then red = max: 1 -> 0.8, 3 -> 0.9
    assert greedy(rel, sims, 4, 0.0) == [0, 2, 1, 3]


def test_an_exact_duplicate_is_demoted():
    rel = f32(1.0, 1.0, 0.8)  # slot 1 is a copy of slot 0 and as relevant
    sims = np.array([[1.0, 1.0, 0.2], [1.0, 1.0, 0.2], [0.2, 0.2, 1.0]], np.float32)
    assert greedy(rel, sims, 3, 0.5) == [0, 2, 1]
    assert greedy(rel, sims, 3, 1.0) == [0, 1, 2]


def test_ties_go_to_the_lower_slot_and_signed_zeros_tie():
    rel = f32(0.0, -0.0, 0.5, 0.5)
    assert greedy(rel, np.zeros((4, 4)), 4, 1.0) == [2, 3, 0, 1]
    rel = f32(-0.0, 0.0)
    assert greedy(rel, np.zeros((2, 2)), 2, 1.0) == [0, 1]
    assert order_key(f32(-0.0))[0] == order_key(f32(0.0))[0]


def test_nan_ranks_first_and_nans_tie():
    rel = f32(INF, NAN, 1.0, NAN)
    assert greedy(rel, np.zeros((4, 4)), 4, 1.0) == [1, 3, 0, 2]
    k = order_key(f32(-INF, -1, 0, 1, INF, NAN, -NAN))
    assert list(np.argsort(k[:5], kind="stable")) == [0, 1, 2, 3, 4] and k[5] == k[6] > k[4]
    # a later pick whose red is NaN (every sim NaN) has value NaN and ranks first
    rel = f32(1.0, 0.5, 0.9)
    sims = np.zeros((3, 3), np.float32)
    sims[1, 0] = NAN
    assert greedy(rel, sims, 3, 0.5) == [0, 1, 2]


# lambda, and (rel, red) of two slots whose values tie under the header's expression (every operation rounded to fp32), while
# a fused multiply-add fma(lambda, rel, -fp32((1 - lambda) * red)) ranks the second slot above the first.  red are multiples of
# 1/128, the sims of one-row 1-bit pages; test_gpu_mmr.py runs the same numbers on the device.
FMA_TIE = (np.float32(0.6369617), (np.float32(0.040973525), np.float32(65 / 128)), (np.float32(-0.097062), np.float32(34 / 128)))


def test_value_is_the_headers_fp32_expression():
    lam, (rel1, red1), (rel2, red2) = FMA_TIE
    one_m = np.float32(1) - lam

    def header(rel, red):
        return (lam * rel) - (one_m * red)

    def fused(rel, red):  # lambda * rel exact in float64, one rounding at the end
        return np.float32(np.float64(lam) * np.float64(rel) - np.float64(one_m * red))

    assert header(rel1, red1) == header(rel2, red2)  # a tie: the lower slot
    assert fused(rel2, red2) > fused(rel1, red1)  # contracted, the order flips
    rel = f32(10.0, rel1, rel2)
    sims = np.zeros((3, 3), np.float32)
    sims[1, 0], sims[2, 0] = red1, red2
    assert greedy(rel, sims, 3, float(lam)) == [0, 1, 2]
    sims[1, 0] = np.nextafter(red1, np.float32(1))  # a slightly larger red of slot 1 hands the tie to slot 2
    assert greedy(rel, sims, 3, float(lam)) == [0, 2, 1]


def test_duplicate_and_unused_slots():
    ids = np.array([3, -1, 7, 3, 99, 2, 7], np.int64)
    assert valid_slots(ids, 10).tolist() == [True, False, True, False, False, True, False]
    rel = f32(0.1, 5.0, 0.3, 9.0, 9.0, 0.2, 9.0)
    assert greedy(rel, np.zeros((7, 7)), 7, 0.5, valid_slots(ids, 10)) == [2, 5, 0]


def test_empty_pages_have_zero_similarity():
    rng = np.random.default_rng(0)
    for kind in ("bf16", "fp8", "int8", "bits"):
        a, e = quantise(rng.standard_normal((5, 128)).astype(np.float32), kind), quantise(np.zeros((0, 128), np.float32), kind)
        assert page_sum(a, e, kind) == 0 and page_sum(e, a, kind) == 0
        assert float(sim_value(page_sum(e, a, kind), 0, 1.0, kind)) == 0.0
        sims = page_sims([a, e], np.array([0, 1]), kind, 1.0)
        assert sims[0, 1] == 0 and sims[1, 0] == 0


def test_relevance_is_mean_per_token():
    assert relevance(f32(3.0, -1.0), 2).tolist() == [1.5, -0.5]
    assert relevance(f32(3.0), 0).tolist() == [3.0]


@pytest.mark.parametrize("kind", ["bf16", "fp8", "int8", "bits"])
def test_page_sims_against_a_scalar_loop(kind):
    rng = np.random.default_rng({"bf16": 1, "fp8": 2, "int8": 3, "bits": 4}[kind])
    lens = [0, 1, 3, 7, 2]
    raw = [rng.standard_normal((n, 128)).astype(np.float32) for n in lens]
    raw[3][4] = raw[2][1]  # a shared row
    pages = [quantise(x, kind) for x in raw]
    scale = {"bf16": 1.0, "fp8": 1 / 4096, "int8": 1 / 127 ** 2, "bits": 1 / 128}[kind]
    ids = np.array([1, 2, -1, 3, 4, 0, 2], np.int64)
    got = page_sims(pages, ids, kind, scale)
    valid = valid_slots(ids, len(pages))

    def dot(x, y):
        if kind == "bits":
            return 128 - sum(bin(int(a) ^ int(b)).count("1") for a, b in zip(x, y))
        if kind == "int8":
            return sum(int(a) * int(b) for a, b in zip(x, y))
        return sum(float(a) * float(b) for a, b in zip(x, y))

    for j in range(len(ids)):
        for s in range(len(ids)):
            if not (valid[j] and valid[s]):
                assert np.isnan(got[j, s])
                continue
            dj, ds = pages[ids[j]], pages[ids[s]]
            S = sum(max(dot(r, c) for c in ds) for r in dj) if len(dj) and len(ds) else 0
            if kind in ("int8", "bits"):
                want = np.float32(0) if not len(dj) else np.float32(np.float32(S) * np.float32(scale)) / np.float32(len(dj))
                assert got[j, s] == want, (j, s)
            else:
                want = S * scale / len(dj) if len(dj) else 0.0
                assert abs(got[j, s] - want) <= 1e-9 * max(1.0, abs(want)), (j, s)
    # a page against itself covers itself completely: every row's max is its own norm (float kinds: |row|^2)
    if kind == "bits":
        assert got[1, 1] == np.float32(1.0)
