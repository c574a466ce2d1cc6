"""The near-duplicate oracle (tests/duplicates_oracle.py) against brute force on small random and planted corpora, and the
pair canonicalisation the index uses (morphik_core_b200.index.candidate_pairs) against the oracle's."""
import numpy as np
import pytest
import torch

from duplicates_oracle import canonical_pairs, collapsed_topk, edges, pair_sims, union_find_labels
from mmr_oracle import quantise_rows
from morphik_core_b200.index import candidate_pairs


def _unit(rng, n):
    x = rng.standard_normal((n, 128)).astype(np.float32)
    return x / np.maximum(np.linalg.norm(x, axis=1, keepdims=True), 1e-9)


def _components(n, edge_list, allowed):
    """Brute force: flood fill from every allowed page, the label the smallest page reached."""
    adj = {p: set() for p in range(n)}
    for x, y in edge_list:
        adj[x].add(y)
        adj[y].add(x)
    out = np.full(n, -1, np.int64)
    for p in range(n):
        if allowed is not None and not allowed[p]:
            continue
        seen, todo = {p}, [p]
        while todo:
            for y in adj[todo.pop()]:
                if y not in seen:
                    seen.add(y)
                    todo.append(y)
        out[p] = min(seen)
    return out


@pytest.mark.parametrize("seed", range(6))
def test_labels_are_the_smallest_page_of_each_component(seed):
    rng = np.random.default_rng(seed)
    n, m = 60, 70
    a, b = rng.integers(0, n, m), rng.integers(0, n, m)
    sab, sba = rng.random(m), rng.random(m)
    sab[:5] = np.nan
    allowed = rng.random(n) > 0.2 if seed % 2 else None
    e = edges(a, b, sab, sba, 0.4, allowed)
    assert all(min(sab[i], sba[i]) >= 0.4 for i in range(m) if (a[i], b[i]) in e and a[i] != b[i])
    assert not any(np.isnan(sab[i]) and (a[i], b[i]) in e for i in range(5))
    assert np.array_equal(union_find_labels(n, e, allowed), _components(n, e, allowed))


def test_dup_is_the_smaller_direction_and_a_subset_is_not_a_duplicate():
    rng = np.random.default_rng(3)
    big = _unit(rng, 40)
    pages = [quantise_rows(p, "bf16") for p in (big, big[:10], big.copy())]
    sab, sba = pair_sims(pages, [1, 0], [0, 2], "bf16", 1.0)
    assert sab[0] == pytest.approx(1.0, abs=1e-2) and sba[0] < 0.6  # the subset is covered (bf16 norms), the big page is not
    assert edges([1], [0], sab[:1], sba[:1], 0.9) == []
    assert edges([0], [2], sab[1:], sba[1:], 0.9) == [(0, 2)]


@pytest.mark.parametrize("kind", ["bf16", "int8", "bits"])
def test_pair_sims_against_brute_force(kind):
    rng = np.random.default_rng(7)
    pages = [quantise_rows(_unit(rng, n), kind) for n in (0, 1, 5, 33, 70)]
    a, b = np.array([0, 1, 2, 3, 4, 4]), np.array([4, 2, 3, 4, 1, 4])
    sab, sba = pair_sims(pages, a, b, kind, 1.0)
    for i in range(len(a)):
        x, y = pages[a[i]].astype(np.float64), pages[b[i]].astype(np.float64)
        if kind == "bits":
            x = np.unpackbits(pages[a[i]], axis=1).astype(np.float64) * 2 - 1
            y = np.unpackbits(pages[b[i]], axis=1).astype(np.float64) * 2 - 1
        for got, p, q in ((sab[i], x, y), (sba[i], y, x)):
            if len(p) == 0 or len(q) == 0:
                assert got == 0
                continue
            m = p @ q.T
            if kind == "bits":
                m = (m + 128) / 2  # 128 - hamming from the +-1 dot
            assert got == pytest.approx(m.max(axis=1).sum() / len(p), rel=1e-6)


def test_canonical_pairs_and_the_index_agree():
    rng = np.random.default_rng(1)
    src = [3, 9, 4, 0]
    ti = torch.as_tensor(rng.integers(-1, 12, size=(4, 6)), dtype=torch.int64)
    ti[1, 2] = 9  # the source itself
    a, b = candidate_pairs([(src[:2], ti[:2]), (src[2:], ti[2:])], 3, "cpu")
    want_a, want_b = [], []
    for s, row in zip(src, ti.tolist()):
        kept = [c for c in row if c >= 0 and c != s][:3]
        want_a += [s] * len(kept)
        want_b += kept
    wa, wb = canonical_pairs(want_a, want_b)
    assert a.tolist() == wa.tolist() and b.tolist() == wb.tolist()
    assert all(x < y for x, y in zip(a.tolist(), b.tolist()))
    e = candidate_pairs([], 3, "cpu")
    assert e[0].numel() == 0 and e[1].numel() == 0


def test_collapsed_topk_against_brute_force():
    rng = np.random.default_rng(5)
    n = 40
    scores = rng.integers(0, 10, n).astype(np.float32)  # ties
    labels = rng.integers(0, 8, n)
    labels[::7] = -1
    got = collapsed_topk(scores, labels, 5)
    best = {}
    for p in range(n):
        if labels[p] < 0:
            continue
        cur = best.get(labels[p])
        if cur is None or (scores[p], -p) > (scores[cur], -cur):
            best[labels[p]] = p
    want = sorted(best.values(), key=lambda p: (-scores[p], p))[:5]
    assert got == want
