"""CPU checks of the explain oracle (tests/explain_oracle.py): brute force on small cases, the lowest-row tie rule, the
fill values of empty pages, and that its per-token maxima add up to the oracle's MaxSim scores."""
import itertools

import numpy as np
import pytest

from explain_oracle import KINDS, maxsim_explain_np, quantise
from oracle import maxsim_oracle as orc


def _data(seed, lens, t):
    rng = np.random.default_rng(seed)
    rows = rng.standard_normal((int(sum(lens)), 128)).astype(np.float32)
    rows /= np.linalg.norm(rows, axis=1, keepdims=True)
    q = rng.standard_normal((t, 128)).astype(np.float32)
    q /= np.linalg.norm(q, axis=1, keepdims=True)
    return q, rows, orc.page_offsets(lens)


@pytest.mark.parametrize("kind", KINDS)
def test_brute_force(kind):
    q, rows, off = _data(1, [3, 0, 1, 7], 5)
    qq, rr = quantise(q, kind), quantise(rows, kind)
    best, arg, maps = maxsim_explain_np(qq, rr, off, kind)
    for p, t in itertools.product(range(len(off) - 1), range(q.shape[0])):
        vals = []
        for r in range(off[p], off[p + 1]):
            if kind == "bits":
                vals.append(128 - int(np.bitwise_count(qq[t] ^ rr[r]).sum()))
            elif kind == "int8":
                vals.append(int(sum(int(a) * int(b) for a, b in zip(qq[t], rr[r]))))
            else:
                vals.append(float(np.dot(qq[t].astype(np.float64), rr[r].astype(np.float64))))
        assert maps[p].shape == (q.shape[0], off[p + 1] - off[p])
        if not vals:
            assert best[p, t] == 0 and arg[p, t] == -1
            continue
        np.testing.assert_allclose(maps[p][t], vals, rtol=1e-12, atol=1e-12)
        assert best[p, t] == max(vals)
        assert arg[p, t] == vals.index(max(vals))


@pytest.mark.parametrize("kind", KINDS)
def test_ties_report_the_lowest_row(kind):
    q, rows, off = _data(2, [9], 3)
    rows[[4, 6, 8]] = rows[2]
    q[:] = rows[2]  # every token's max is row 2 and its three copies
    best, arg, maps = maxsim_explain_np(quantise(q, kind), quantise(rows, kind), off, kind)
    assert (arg[0] == 2).all()
    assert (maps[0][:, [4, 6, 8]] == best[0][:, None]).all()
    same = np.repeat(rows[:1], 5, axis=0)
    best, arg, _ = maxsim_explain_np(quantise(q, kind), quantise(same, kind), orc.page_offsets([5]), kind)
    assert (arg[0] == 0).all()


@pytest.mark.parametrize("kind", KINDS)
def test_sums_equal_the_maxsim_oracle(kind):
    lens = [0, 1, 31, 32, 33, 70]
    q, rows, off = _data(3, lens, 37)
    qq, rr = quantise(q, kind), quantise(rows, kind)
    best, arg, _ = maxsim_explain_np(qq, rr, off, kind)
    if kind == "bits":
        want = orc.binary_maxsim_np(qq, rr, off)[1]
        assert np.array_equal(best.sum(axis=1), want)
    elif kind == "int8":
        assert np.array_equal(best.sum(axis=1), orc.int8_maxsim_np(qq, rr, off))
    else:
        np.testing.assert_allclose(best.sum(axis=1), orc.float_maxsim_np(qq, rr, off), rtol=1e-6)
    assert (arg[0] == -1).all() and (best[0] == 0).all()  # the empty page
    assert ((arg[1:] >= 0) & (arg[1:] < np.asarray(lens[1:])[:, None])).all()
