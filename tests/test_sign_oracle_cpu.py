"""The numpy oracle of the asymmetric sign stage (tests/sign_oracle.py) checked on its own, without a GPU: the sign rule of
every dtype against the float signs of oracle/value_rules.py's packed values, every edge of the query quantiser, the
2 q8 / c_t form of the scan against the +-1 dot product, empty pages, padding tokens and the tie order."""
import numpy as np
import pytest
import torch

import sign_oracle as so
from oracle import value_rules as vr


def _bits(x):
    return torch.from_numpy(np.ascontiguousarray(x, dtype=np.float32).view(np.int32))


def _special_rows():
    rng = np.random.default_rng(0)
    specials = np.array([0.0, -0.0, np.nan, -np.nan, np.inf, -np.inf, 1e-40, -1e-40, 1e-3, -1e-3, 3e38, -3e38, 0.004, -0.004,
                         1.0, -1.0], dtype=np.float32)
    x = rng.standard_normal((64, 128)).astype(np.float32) * rng.choice([1e-3, 0.05, 1.0, 500.0], size=(64, 1))
    x[:8] = np.resize(specials, (8, 128))
    return x


def _decoded(dtype, packed):
    """The float value of every packed element (bf16 widened, int8 as is, e4m3 decoded)."""
    if dtype == "bf16":
        return (packed.view("<u2").astype(np.uint32) << 16).view(np.float32).reshape(-1, 128)
    if dtype == "int8":
        return packed.view(np.int8).astype(np.float32).reshape(-1, 128)
    return torch.from_numpy(packed.copy()).view(torch.float8_e4m3fn).float().numpy().reshape(-1, 128)


def test_sign_rule_is_the_float_sign_of_the_packed_value():
    x = _special_rows()
    for dtype, scale in (("bf16", 1.0), ("int8", 127.0), ("fp8", 64.0)):
        packed = vr.packed_bytes(dtype, _bits(x), scale).numpy()
        got = so.pack_bits(so.sign_bits(dtype, packed))
        want = vr.sign_bytes(_bits(_decoded(dtype, packed))).numpy()  # bit = float32(value) > 0
        np.testing.assert_array_equal(got, want, err_msg=dtype)


def test_sign_rule_edges():
    bf = np.array([0x0000, 0x8000, 0x7FFF, 0xFFFF, 0x7F80, 0xFF80, 0x0001, 0x8001, 0x3F80, 0x7F81], dtype="<u2")
    want = [0, 0, 0, 0, 1, 0, 1, 0, 1, 0]
    assert so.sign_bits("bf16", np.resize(bf, 128).view(np.uint8))[0, :10].tolist() == [bool(w) for w in want]
    i8 = np.array([0, 1, 127, -1, -127], dtype=np.int8)
    assert so.sign_bits("int8", np.resize(i8, 128).view(np.uint8))[0, :5].tolist() == [False, True, True, False, False]
    f8 = np.array([0x00, 0x80, 0x7F, 0xFF, 0x7E, 0x01, 0x81, 0xFE], dtype=np.uint8)
    assert so.sign_bits("fp8", np.resize(f8, 128))[0, :8].tolist() == [False, False, False, False, True, True, False, False]


def test_pack_bits_is_msb_first():
    b = np.zeros((1, 128), dtype=bool)
    b[0, 0] = b[0, 9] = b[0, 127] = True
    r = so.pack_bits(b)
    assert r.shape == (1, 16) and r[0, 0] == 0x80 and r[0, 1] == 0x40 and r[0, 15] == 0x01
    np.testing.assert_array_equal(so.unpack_bits(r), b)


def test_quantiser_edges():
    s = 2.0
    x = np.zeros((1, 128), dtype=np.float32)
    vals = [1.25, 1.75, -1.25, -1.75, 0.25, -0.25, 31.75, 31.5, 32.0, -32.0, -100.0, np.nan, np.inf, -np.inf, -0.0, 0.75]
    want = [2, 4, -2, -4, 0, 0, 63, 63, 63, -63, -63, 0, 63, -63, 0, 2]  # 2.5 -> 2, 3.5 -> 4 (ties to even), +-63 clamp
    x[0, :len(vals)] = vals
    q = so.quantise_query(x, s)
    assert q[0, :len(vals)].tolist() == want and q.dtype == np.int64
    assert (q[0, len(vals):] == 0).all()
    # the product is rounded in float32 before rint: 0.1f * 25 is 2.5000000372..., not a tie
    assert so.quantise_query(np.full((1, 128), 0.1, np.float32), 25.0)[0, 0] == int(np.rint(np.float32(0.1) * np.float32(25.0)))


def test_operands_give_the_pm1_dot_product():
    rng = np.random.default_rng(1)
    q8 = rng.integers(-63, 64, size=(40, 128))
    q8[0] = 63
    q8[1] = -63
    bits = rng.integers(0, 2, size=(50, 128)).astype(bool)
    a, c = so.operands(q8)
    assert np.abs(a).max() <= 126  # fits int8
    got = a @ bits.astype(np.int64).T + c[:, None]
    want = q8 @ np.where(bits, 1, -1).T
    np.testing.assert_array_equal(got, want)
    # a padding token (all zero) contributes 0 through both operands
    a0, c0 = so.operands(np.zeros((1, 128), np.int64))
    assert (a0 == 0).all() and c0[0] == 0


def test_scores_empty_pages_padding_rows_and_empty_queries():
    rng = np.random.default_rng(2)
    lens = [3, 0, 33, 1, 0, 64]
    ps = so.page_starts(lens)
    bits = rng.integers(0, 2, size=(int(ps[-1]), 128)).astype(bool)
    for p, n in enumerate(lens):  # padding rows repeat the last true row; rows past it must not count anyway
        if n:
            bits[ps[p] + n:ps[p + 1]] = ~bits[ps[p] + n - 1]
    q8s = [rng.integers(-63, 64, size=(t, 128)) for t in (5, 0, 1)]
    s = so.scores(q8s, bits, lens)
    assert s.shape == (3, 6) and (s[:, [1, 4]] == 0).all() and (s[1] == 0).all()
    pm = np.where(bits, 1, -1)
    for q, q8 in enumerate(q8s):
        for p, n in enumerate(lens):
            if n and len(q8):
                want = sum(max(int(q8[t] @ pm[ps[p] + r]) for r in range(n)) for t in range(len(q8)))
                assert s[q, p] == want


def test_probe_corpus_decodes_q8():
    rng = np.random.default_rng(3)
    q8 = rng.integers(-63, 64, size=(20, 128))
    q8[0], q8[1], q8[2] = 63, -63, 0
    bits = so.probe_bits()
    assert bits.sum() == 128 and not bits[0].any()
    padded = np.repeat(bits, 32, axis=0)  # single-row pages, padding rows repeat the row
    s = so.scores(list(q8[:, None, :]), padded, [1] * 129)
    np.testing.assert_array_equal(so.probe_q8(s), q8)
    # brute force: page 1 + i scores -sum q8 + 2 q8_i
    np.testing.assert_array_equal(s[:, 1:], -q8.sum(axis=1, keepdims=True) + 2 * q8)
    s[0, 5] += 1
    with pytest.raises(ValueError):
        so.probe_q8(s)


@pytest.mark.parametrize("scale", [127.0, 32.0, 512.0, 1.0, 0.75])
def test_tie_inputs_are_ties(scale):
    x = so.tie_inputs(scale)
    assert x.dtype == np.float32
    y = x * np.float32(scale)
    assert set(y.tolist()) <= {k + 0.5 for k in range(-64, 64)} and len(set(y.tolist())) == len(x)
    if scale in (32.0, 512.0, 1.0):  # a power of two: every k has its tie
        assert len(x) == 128
    # brute force over the float32 bit patterns within 4 ulps of (k + 0.5) / scale: a k without a returned x has no tie
    found = set(y.tolist())
    for k in range(-64, 64):
        x0 = np.array([(k + 0.5) / scale], dtype=np.float32).view(np.int32)[0]
        near = (x0 + np.arange(-4, 5, dtype=np.int32)).view(np.float32)
        assert bool((near * np.float32(scale) == np.float32(k + 0.5)).any()) == ((k + 0.5) in found), k
    # the quantiser rounds every tie to the even neighbour, then clamps
    q = so.quantise_query(np.resize(x, (len(x) + 127) // 128 * 128).reshape(-1, 128), scale).reshape(-1)[:len(x)]
    lo = np.floor(y)
    np.testing.assert_array_equal(q, np.clip(np.where(lo % 2 == 0, lo, lo + 1), -63, 63).astype(np.int64))


def test_topk_order_and_masks():
    s = np.array([5, 7, 7, -1, 5, 7, 0], dtype=np.int64)
    assert so.topk(s, 10) == [1, 2, 5, 0, 4, 6, 3]  # score DESC, page id ASC
    assert so.topk(s, 2) == [1, 2]
    words = np.array([0b1011001], dtype=np.uint32)  # pages 0, 3, 4, 6
    allowed = so.mask_allowed(words, 7)
    assert allowed.tolist() == [True, False, False, True, True, False, True]
    assert so.topk(s, 3, allowed) == [0, 4, 6]
