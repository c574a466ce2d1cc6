"""The I32 sum rule of oracle.scoring (int64 sums clamped to +-(2^31 - 1)) against hand-worked boundary cases.

An int8 token scores at most 128 * 127 * 127 = 2 064 512 against a +-127 row, or 128 * 127 * 128 = 2 080 768 against a
-128 row, so the first query lengths whose sum passes 2^31 - 1 are 1041 and 1033 tokens.
"""
import numpy as np

from oracle import maxsim_oracle as orc
from oracle.scoring import I32_SUM_BOUND, i32_reported, i32_sum

M = 2147483647
TOKEN_127 = 128 * 127 * 127
TOKEN_128 = 128 * 127 * 128


def test_token_maxima():
    assert TOKEN_127 == 2_064_512 and TOKEN_128 == 2_080_768 and I32_SUM_BOUND == M


# (tokens, token score, exact sum, what int32 would wrap it to, the clamped sum)
ROWS = [
    (1040, TOKEN_127, 2_147_092_480, 2_147_092_480, 2_147_092_480),
    (1041, TOKEN_127, 2_149_156_992, -2_145_810_304, M),
    (1041, -TOKEN_127, -2_149_156_992, 2_145_810_304, -M),
    (2080, TOKEN_127, 4_294_184_960, -782_336, M),
    (2081, TOKEN_127, 4_296_249_472, 1_282_176, M),
    (1032, TOKEN_128, 2_147_352_576, 2_147_352_576, 2_147_352_576),
    (1033, TOKEN_128, 2_149_433_344, -2_145_533_952, M),
    (1033, -TOKEN_128, -2_149_433_344, 2_145_533_952, -M),
]


def test_boundary_rows():
    for t, tok, exact, wrapped, clamped in ROWS:
        assert t * tok == exact
        assert int(np.int64(exact).astype(np.int32)) == wrapped  # what an int32 accumulator leaves
        assert int(i32_sum(exact)) == clamped, (t, tok)


def test_bound_and_one_past():
    sums = np.asarray([M - 1, M, M + 1, -M + 1, -M, -M - 1, 1 << 40, -(1 << 40), 0], np.int64)
    assert i32_sum(sums).tolist() == [M - 1, M, M, -M + 1, -M, -M, M, -M, 0]
    assert i32_sum(sums).dtype == np.int64


def test_reported_scores():
    """float32 rounds both M - 1 and M to 2^31: only the order can tell them apart.  Below 2^24 the report is exact."""
    scale = 1.0 / (127.0 * 127.0)
    got = i32_reported(np.asarray([M - 1, M, M + 5, -M - 5, 2_147_092_480, 12345], np.int64), scale)
    assert got.dtype == np.float32
    f = np.float32
    assert got.tolist() == [f(2.0 ** 31) * f(scale), f(2.0 ** 31) * f(scale), f(2.0 ** 31) * f(scale),
                            f(-(2.0 ** 31)) * f(scale), f(2_147_092_480) * f(scale), f(12345) * f(scale)]
    assert i32_reported([3], 1.0).tolist() == [3.0]


def test_the_int64_oracle_reaches_the_bound():
    """The int8 oracle keeps the 1041-token sum exact; only the rule clamps it."""
    q = np.full((1041, 128), 127, np.int8)
    rows = np.concatenate([np.full((1, 128), 127, np.int8), np.full((1, 128), -127, np.int8), np.full((1, 128), -128, np.int8)])
    got = orc.int8_maxsim_c(q, rows, orc.page_offsets([1, 1, 1]))
    assert got.tolist() == [1041 * TOKEN_127, -1041 * TOKEN_127, -1041 * TOKEN_128]
    assert i32_sum(got).tolist() == [M, -M, -M]
    got = orc.int8_maxsim_c(-q[:1033], rows[2:], orc.page_offsets([1]))
    assert got.tolist() == [1033 * TOKEN_128] and i32_sum(got).tolist() == [M]
