"""The value rules of the oracle (no GPU): quantisers and top-k order on the inputs where conversions and comparisons go
wrong -- rounding ties, signed zeros, subnormals, saturation, infinities and NaN.

The torch restatements in oracle/value_rules.py (what tests/test_gpu_quantisers.py runs on the GPU over every float32 bit
pattern) are tied here to the numpy oracle, on a 2^20-pattern sample plus every special class.
"""
import numpy as np
import pytest

from oracle import maxsim_oracle as orc

torch = pytest.importorskip("torch")
from oracle import value_rules as vr  # noqa: E402

F32 = np.float32


def special_patterns() -> np.ndarray:
    """float32 bit patterns of every special class, both signs: zeros, subnormals (smallest, largest, ties), the smallest
    normal, the largest finite, infinities, quiet and signalling NaNs with several payloads, bf16 / e4m3 / int8 rounding ties
    and their neighbours."""
    mags = [0x00000000, 0x00000001, 0x00000002, 0x00007FFF, 0x00008000, 0x00008001, 0x00018000, 0x007FFFFF,
            0x00800000, 0x00800001, 0x7F7FFFFF, 0x7F7F8000, 0x7F7F7FFF, 0x7F800000, 0x7F800001, 0x7F800002,
            0x7FBFFFFF, 0x7FC00000, 0x7FC00001, 0x7FFFFFFF, 0x3F800000, 0x3F808000, 0x3F818000, 0x3F807FFF, 0x3F808001]
    vals = []
    for v in (0.5, 1.5, 2.5, 126.5, 127.4999, 127.5, 128.0, 1e6, 448.0, 464.0, 479.9, 480.0, 1.0625, 1.1875, 2.0 ** -7,
              2.0 ** -10, 3 * 2.0 ** -11, 2.0 ** -9 * 1.5):
        for s in (1.0, 1 / 64, 1 / 127, 1 / 48):  # ties at the library's scales
            vals.append(np.asarray(v * s, F32).view(np.uint32))
            vals.append(np.nextafter(np.asarray(v * s, F32), F32(np.inf)).view(np.uint32))
            vals.append(np.nextafter(np.asarray(v * s, F32), F32(0)).view(np.uint32))
    m = np.asarray(mags + [int(v) for v in vals], dtype=np.uint32)
    return np.concatenate([m, m | np.uint32(0x80000000)])


def sample_patterns(n=1 << 20, seed=1) -> np.ndarray:
    rng = np.random.default_rng(seed)
    r = rng.integers(0, 1 << 32, size=n, dtype=np.uint64).astype(np.uint32)
    return np.concatenate([r, special_patterns()])


def _f(bits):
    return np.asarray(bits, np.uint32).view(F32)


def _t(bits):
    return torch.from_numpy(np.asarray(bits, np.uint32).view(np.int32).copy())


# ------------------------------------------------------------------------------------------------ restatement == oracle
def test_bf16_restatement_equals_oracle():
    b = sample_patterns()
    want = orc.bf16_round_np(_f(b)).view(np.uint32) >> 16
    assert np.array_equal(vr.bf16_bits(_t(b)).numpy(), want.astype(np.int64))


@pytest.mark.parametrize("scale", [127.0, 1.0])
def test_int8_restatement_equals_oracle(scale):
    b = sample_patterns()
    assert np.array_equal(vr.int8_codes(_t(b), scale).numpy(), orc.quantize_int8_np(_f(b), scale))


@pytest.mark.parametrize("scale", [64.0, 48.0])
def test_e4m3_restatement_equals_oracle(scale):
    b = sample_patterns()
    assert np.array_equal(vr.e4m3_codes(_t(b), scale).numpy(), orc.quantize_e4m3_np(_f(b), scale))


def test_sign_restatement_equals_oracle():
    b = sample_patterns()
    b = b[: len(b) // 128 * 128]
    assert np.array_equal(vr.sign_bytes(_t(b)).numpy(), orc.sign_pack_np(_f(b).reshape(-1, 128)))


# ------------------------------------------------------------------------------------------------ the rules themselves
def test_bf16_rule_on_special_values():
    x = _f([0x3F808000, 0x3F818000, 0x3F808001, 0x7F7FFFFF, 0xFF7FFFFF, 0x00000001, 0x00008000, 0x80008000,
            0x7FC00000, 0xFFC00001, 0x7F800001])
    got = orc.bf16_round_np(x).view(np.uint32) >> 16
    # ties to even (down, up), above a tie, overflow to +-inf, subnormals kept (and a subnormal tie to even), NaN canonical
    assert got.tolist() == [0x3F80, 0x3F82, 0x3F81, 0x7F80, 0xFF80, 0x0000, 0x0000, 0x8000, 0x7FFF, 0x7FFF, 0x7FFF]


def test_int8_rule_nan_inf_ties_and_saturation():
    x = np.asarray([np.nan, -np.nan, np.inf, -np.inf, 0.5, 1.5, 2.5, -0.5, -2.5, 126.5, 127.5, 1e30, -0.0,
                    1e-45], F32)
    got = orc.quantize_int8_np(x, 1.0)
    assert got.tolist() == [0, 0, 127, -127, 0, 2, 2, 0, -2, 126, 127, 127, 0, 0]
    nan_neg = np.asarray([0xFFFFFFFF, 0xFF800001], np.uint32).view(F32)
    assert orc.quantize_int8_np(nan_neg, 127.0).tolist() == [0, 0]  # NaN is 0 whatever its sign bit, not -127
    assert orc.quantize_int8_np(np.asarray([1e38], F32), 127.0).tolist() == [127]  # fp32 product overflows to inf


def test_e4m3_rule_nan_inf_ties_and_saturation():
    x = np.asarray([np.nan, np.inf, -np.inf, 448.0, 464.0, 480.0, 1e30, -0.0, 0.0, 1.0625, 1.1875, 2.0 ** -10,
                    3 * 2.0 ** -10, 2.0 ** -11], F32)
    got = orc.quantize_e4m3_np(x, 1.0)
    # 1.0625 ties to 1.0 (even code 0x38), 1.1875 ties to 1.25 (0x3a); 2^-10 ties to 0, 3*2^-10 to 2^-8 (code 2),
    # 2^-11 below the smallest half-subnormal -> 0
    assert got.tolist() == [0x7F, 0x7E, 0xFE, 0x7E, 0x7E, 0x7E, 0x7E, 0x80, 0x00, 0x38, 0x3A, 0x00, 0x02, 0x00]
    nan_neg = np.asarray([0xFFC00000, 0xFFFFFFFF], np.uint32).view(F32)
    assert orc.quantize_e4m3_np(nan_neg, 64.0).tolist() == [0x7F, 0x7F]  # the device drops a NaN's sign


def _e4m3_float64_rule(x, scale):
    """The rule the oracle used before: the product x * scale taken exactly (float64), then one rounding to e4m3."""
    y = np.asarray(x, F32).astype(np.float64) * scale
    a = np.minimum(np.abs(y), 448.0)
    tab = orc._E4M3
    hi = np.clip(np.searchsorted(tab, a, side="left"), 0, len(tab) - 1)
    lo = np.maximum(hi - 1, 0)
    pick_hi = (tab[hi] - a < a - tab[lo]) | ((tab[hi] - a == a - tab[lo]) & (hi % 2 == 0))
    return np.where(pick_hi, hi, lo).astype(np.uint8) | (np.signbit(y).astype(np.uint8) << 7)


def test_e4m3_multiplies_in_float32():
    """With a scale that is not a power of two the fp32 product can land exactly on an e4m3 tie that the exact product
    misses: the library rounds twice (fp32 product, then e4m3), and so does the oracle."""
    x = _f(sample_patterns(1 << 20, seed=7))
    x = x[np.isfinite(x)]
    diff = np.flatnonzero(_e4m3_float64_rule(x, 48.0) != orc.quantize_e4m3_np(x, 48.0))
    assert len(diff) > 0  # the two rules are distinguishable on this sample ...
    tab = orc._E4M3
    for i in diff:  # ... and wherever they differ, the fp32 product sits exactly on a tie (or on 464, saturated by both)
        y32 = abs(np.float64(x[i] * F32(48.0)))
        j = np.searchsorted(tab, y32)
        assert j < len(tab) and tab[j] - y32 == y32 - tab[j - 1], (x[i], y32)


def test_finite_power_of_two_results_unchanged():
    """The new rules change nothing on finite data at a power-of-two scale: int8 and e4m3 of Gaussian rows equal the
    formulations the oracle used before."""
    rng = np.random.default_rng(3)
    x = (rng.standard_normal((4096, 128)) * rng.choice([1e-3, 0.1, 1.0, 10.0], size=(4096, 1))).astype(F32)
    assert np.array_equal(orc.quantize_int8_np(x, 127.0), np.clip(np.rint(x * F32(127.0)), -127, 127).astype(np.int8))
    assert np.array_equal(orc.quantize_e4m3_np(x, 64.0), _e4m3_float64_rule(x, 64.0))
    bf = orc.bf16_round_np(x).view(np.uint32)
    u = x.view(np.uint32).astype(np.uint64)
    assert np.array_equal(bf, (((u + 0x7FFF + ((u >> 16) & 1)) >> 16) << 16).astype(np.uint32))


# ------------------------------------------------------------------------------------------------ top-k order
def test_topk_order_nan_first_and_signed_zeros_tie():
    neg_nan = np.uint32(0xFFFFFFFF).view(F32)
    s = np.asarray([0.0, -0.0, 1.0, np.nan, -np.inf, np.inf, neg_nan, -0.0, 0.0, -1.0, np.nan], F32)
    vals, ids = orc.topk_np(s, len(s))
    # NaNs (either sign) first and tied (id order), then +inf, 1, the four zeros in id order, -1, -inf
    assert ids.tolist() == [3, 6, 10, 5, 2, 0, 1, 7, 8, 9, 4]
    vals, ids = orc.topk_np(s, 4, allow=np.asarray([True, True, True, False, True, False, False, True, True, True, True]))
    assert ids.tolist() == [10, 2, 0, 1]


def test_rank_desc_np_orders_by_id_not_position():
    s = np.asarray([1.0, 1.0, -0.0, 0.0, np.nan], F32)
    ids = np.asarray([9, 2, 7, 3, 1 << 62], np.int64)
    assert ids[orc.rank_desc_np(s, ids)].tolist() == [1 << 62, 2, 9, 3, 7]


def test_topk_on_int_scores_is_exact_beyond_float32():
    s = np.asarray([(1 << 24) + 1, 1 << 24, (1 << 31) - 1, -(1 << 31) + 1, (1 << 24) + 1], np.int64)
    vals, ids = orc.topk_np(s, 5)
    assert ids.tolist() == [2, 0, 4, 1, 3]
