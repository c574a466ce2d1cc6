"""tests/float_value_oracle.py against the float value rule of include/b200ms.h: hand-worked cases for every clause and a
brute-force scalar loop (plain Python floats, one product and one addition at a time) on random corpora with non-finite
elements."""
import math

import numpy as np
import pytest

import float_value_oracle as fvo
from oracle import maxsim_oracle as orc

INF, NAN = math.inf, math.nan


def same(a, b):
    """Equal values, NaN equal to NaN (+-0 alike)."""
    return np.array_equal(np.asarray(a, np.float64), np.asarray(b, np.float64), equal_nan=True)


def row(**at):
    r = np.zeros(128)
    for k, v in at.items():
        r[int(k[1:])] = v
    return r


# ------------------------------------------------------------------------------------------------ packed values
def test_bf16_values_cover_every_pattern():
    v = fvo.bf16_values(np.arange(65536, dtype=np.uint32).astype(np.uint16))
    assert v[0x3F80] == 1.0 and v[0xBF80] == -1.0 and v[0x7F80] == INF and v[0xFF80] == -INF
    assert v[0x0001] == 2.0 ** -133 and v[0x0080] == 2.0 ** -126 and v[0x7F7F] == float.fromhex("0x1.fep127")
    assert np.isnan(v).sum() == 254  # exponent all ones, mantissa nonzero, both signs
    assert np.isinf(v).sum() == 2
    assert math.copysign(1.0, v[0x8000]) == -1.0


def test_e4m3_values_nan_codes_and_finite_codes():
    codes = np.arange(256, dtype=np.uint8)
    v = fvo.e4m3_values(codes)
    assert np.flatnonzero(np.isnan(v)).tolist() == [0x7F, 0xFF]
    assert v[0x7E] == 448.0 and v[0xFE] == -448.0 and v[0x01] == 2.0 ** -9 and v[0x38] == 1.0
    fin = (codes & 0x7F) != 0x7F
    assert np.array_equal(v[fin], orc.dequantize_e4m3_np(codes[fin]).astype(np.float64))


def test_pack_values_follow_the_pack_rules():
    x = np.array([1.0, -0.0, INF, -INF, NAN, 1e39, 3.0e38, 2.0 ** -140, 1.0 + 2.0 ** -8], np.float32)
    b = fvo.pack_values("bf16", x)
    # 2^-140 is below bf16's least subnormal 2^-133; 1 + 2^-8 is a tie that rounds to the even 1
    assert same(b, [1.0, -0.0, INF, -INF, NAN, INF, float(orc.bf16_round_np(np.float32(3.0e38))), 0.0, 1.0])
    f = fvo.pack_values("fp8", x)  # codes of x * 64: infinities saturate, NaN stays NaN (0x7f)
    assert same(f, [64.0, -0.0, 448.0, -448.0, NAN, 448.0, 448.0, 0.0, 64.0])


# ------------------------------------------------------------------------------------------------ hand-worked cases
def test_similarity_non_finite_arithmetic():
    d = np.stack([row(e0=INF), row(e0=-INF), row(e0=NAN), row(e0=INF, e1=-INF), row(e0=2.0)])
    q = np.stack([row(e0=0.0, e2=1.0), row(e0=3.0), row(e0=-3.0), row(e0=1.0, e1=1.0)])
    want = [[NAN, NAN, NAN, NAN, 0.0],      # 0 * +-inf = NaN, NaN * 0 = NaN
            [INF, -INF, NAN, NAN, 6.0],     # row 3: 3 * inf + 0 * -inf = NaN
            [-INF, INF, NAN, NAN, -6.0],
            [INF, -INF, NAN, NAN, 2.0]]     # row 3: +inf + -inf = NaN
    assert same(fvo.similarities(q, d), want)


def test_products_leave_the_fp32_range():
    big, tiny = 2.0 ** 64, 2.0 ** -75
    cases = [  # (query value, row value, sim)
        (big, big, INF), (-big, big, -INF), (2.0 ** 63, big, 2.0 ** 127),
        (2.0 ** -63, 2.0 ** -64, 2.0 ** -127),              # fp32 subnormal, kept
        (2.0 ** -70, 2.0 ** -79, 2.0 ** -149),              # least fp32 subnormal
        (tiny, tiny, 0.0),                                  # 2^-150: below the least subnormal, to 0
        (1.5 * tiny, tiny, 0.0),                            # 1.5 * 2^-150: toward zero, not up to 2^-149
        (-1.0078125 * tiny, tiny, -0.0),                    # measured on an H100: 0, not -2^-149
        (1.5 * 2.0 ** -74, 2.0 ** -75, 2.0 ** -149),        # measured: 1.5 * 2^-149 gives 2^-149, not the even 2^-148
        (-1.75 * 2.0 ** -74, 2.0 ** -70, -(2.0 ** -144) * 1.75),  # a multiple of 2^-149: exact
        (2.0 ** -100, 2.0 ** -100, 0.0),
    ]
    for a, b, want in cases:
        assert same(fvo.similarities(row(e5=a)[None], row(e5=b)[None])[0, 0], want), (a, b)
    # a finite sum past the fp32 range is +-inf; products past it that cancel do not overflow on their own
    assert fvo.similarities(row(e0=1.0, e1=1.0)[None], row(e0=2.0 ** 127, e1=2.0 ** 127)[None])[0, 0] == INF
    assert fvo.similarities(row(e0=big, e1=-big)[None], row(e0=big, e1=big)[None])[0, 0] == 0.0
    assert fvo.similarities(row(e0=big, e1=-big)[None], row(e0=big, e1=2.0 ** -64)[None])[0, 0] == INF


def test_row_max_is_fmaxf():
    s = np.array([[NAN, 1.0, NAN], [NAN, NAN, NAN], [-INF, NAN, -1.0], [INF, NAN, 5.0], [-0.0, NAN, -INF]])
    assert same(fvo.fmax_rows(s), [1.0, NAN, -1.0, INF, 0.0])


def test_page_score_sums_true_tokens_only():
    d = np.stack([row(e0=INF, e1=1.0)] * 3)  # every row holds +inf
    q = np.stack([row(e0=1.0), row(e0=2.0, e1=1.0)])
    assert fvo.page_score(q, d) == INF
    # the same query with a zero padding token appended scores NaN: what the rule keeps out of the group sum
    assert np.isnan(fvo.page_score(np.vstack([q, np.zeros((1, 128))]), d))
    assert fvo.page_score(q, np.zeros((0, 128))) == 0.0  # a page without rows
    assert np.isnan(fvo.page_score(np.stack([row(e0=1.0), row(e0=-1.0)]), d[:1]))  # +inf + -inf over tokens
    assert fvo.page_score(np.stack([row(e0=-1.0, e1=1.0), row(e0=-2.0, e1=1.0)]), d[:1]) == -INF


def test_zero_pad_clamp_turns_nan_into_zero():
    d = np.stack([row(e0=INF), row(e0=INF)])
    q = np.stack([row(e1=1.0), row(e0=-1.0), row(e0=1.0)])  # maxima NaN, -inf, +inf
    assert same(fvo.token_maxima(q, d), [NAN, -INF, INF])
    assert same(fvo.token_maxima(q, d, clamp=True), [0.0, 0.0, INF])
    assert fvo.page_score(q, d, clamp=True) == INF
    assert np.isnan(fvo.page_score(q, d))
    assert fvo.zero_pad_clamped([3, 5, 5, 0, 2, 7], 3).tolist() == [True, False, False, True, True, False]


def test_fp32_rounding_of_finite_sums():
    q = np.stack([row(e0=1.0, e1=1.0)])
    d = np.stack([row(e0=1.0, e1=2.0 ** -30)])  # 1 + 2^-30 is not an fp32
    assert fvo.similarities(q, d)[0, 0] == 1.0
    assert fvo.page_score(np.stack([row(e0=1.0)] * 3), np.stack([row(e0=float(np.float32(0.1)))])) == float(np.float32(3 * np.float32(0.1)))


# ------------------------------------------------------------------------------------------------ brute force
def scalar_score(q, d, clamp=False):
    """Exact products and an exact sum (math.fsum) in Python floats, rounded to fp32 once; NaN and infinities by hand."""
    def f32(x):  # nearest even in the normal range, toward zero to a multiple of 2^-149 below 2^-126
        if abs(x) < 2.0 ** -126:
            return math.trunc(x / 2.0 ** -149) * 2.0 ** -149
        with np.errstate(over="ignore"):
            return float(np.float32(x))

    def add(terms):
        nan = any(math.isnan(t) for t in terms)
        pinf, ninf = INF in terms, -INF in terms
        if nan or (pinf and ninf):
            return NAN
        if pinf or ninf:
            return INF if pinf else -INF
        return f32(math.fsum(terms))

    if len(d) == 0:
        return 0.0
    maxima = []
    for t in q:
        best = NAN
        for r in d:
            s = add([float(a) * float(b) for a, b in zip(t, r)])  # exact; Python floats: 0 * inf is NaN, as IEEE says
            if not math.isnan(s) and (math.isnan(best) or s > best):
                best = s
        if clamp:
            best = 0.0 if math.isnan(best) else max(best, 0.0)
        maxima.append(best)
    return add(maxima)


@pytest.mark.parametrize("dtype", ["bf16", "fp8"])
def test_oracle_equals_brute_force(dtype):
    rng = np.random.default_rng(11 if dtype == "bf16" else 12)
    specials = np.array([INF, -INF, NAN, 0.0, -0.0, 1e38, -1e38, 2.0 ** -130], np.float32)
    for trial in range(40):
        n_rows, n_tok = int(rng.integers(0, 5)), int(rng.integers(1, 5))
        d = rng.standard_normal((n_rows, 128)).astype(np.float32)
        q = rng.standard_normal((n_tok, 128)).astype(np.float32)
        for m in (d, q):
            k = rng.random(m.shape) < 0.03
            m[k] = rng.choice(specials, size=int(k.sum()))
            m[:, :2] = rng.choice(specials, size=(m.shape[0], 2))  # non-finite values meet zeros and each other
        qv, dv = fvo.pack_values(dtype, q), fvo.pack_values(dtype, d)
        for clamp in (False, True):
            got = fvo.page_score(qv, dv, clamp)
            want = scalar_score(qv, dv, clamp)
            assert same(got, want), (trial, clamp, got, want)


def test_scores_matrix_equals_page_score():
    rng = np.random.default_rng(3)
    pages = [rng.standard_normal((n, 128)) for n in (0, 1, 3)]
    pages[2][:, 4] = INF
    qs = [rng.standard_normal((t, 128)) for t in (1, 2)]
    qs[1][:, 4] = 0.0
    clamp = [False, True, True]
    want = [[fvo.page_score(q, d, c) for d, c in zip(pages, clamp)] for q in qs]
    assert same(fvo.scores(qs, pages, clamp), want)
    assert np.isnan(fvo.scores(qs, pages)[1, 2]) and fvo.scores(qs, pages, clamp)[1, 2] >= 0.0


def test_fast_similarities_equal_the_elementwise_ones():
    """The matrix-product path against one product at a time."""
    rng = np.random.default_rng(8)
    specials = np.array([INF, -INF, NAN, 0.0, -0.0, 2.0 ** 100, 2.0 ** -120])
    for _ in range(20):
        q, d = rng.standard_normal((9, 128)), rng.standard_normal((7, 128))
        for m in (q, d):
            k = rng.random(m.shape) < 0.02
            m[k] = rng.choice(specials, size=int(k.sum()))
        q, d = fvo.pack_values("bf16", q), fvo.pack_values("bf16", d)
        assert same(fvo.similarities(q, d), fvo._similarities_elementwise(q, d))
