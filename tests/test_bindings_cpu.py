"""The Python side of the C-ABI without a GPU: the argument checks every device call makes before it hands a tensor to
libb200ms (queries, allow masks, candidate lists, result buffers), the allow-mask format, the run walk of compaction, the
padded page length and the catalogue record format."""
import dataclasses
import json
import logging
import types

import numpy as np
import pytest
import torch

from morphik_core_b200 import _native as nat
from morphik_core_b200.catalog import PageCatalog, PageRecord
from morphik_core_b200.index import (MaxSimIndex, _check_candidates, _check_device_masks, _check_queries, _host_mask_to_device,
                                     _padded_lens, _runs, _topk_outputs)
from morphik_core_b200.store import _capped_k

CPU = torch.device("cpu")
META = torch.device("meta")  # a tensor on another device, without needing a second one


# ------------------------------------------------------------------ queries
@pytest.mark.parametrize("dtype,code", [(torch.float32, nat.F32), (torch.bfloat16, nat.BF16)])
def test_queries_valid(dtype, code):
    assert _check_queries(torch.zeros((70, 128), dtype=dtype), [32, 38], CPU) == code
    assert _check_queries(torch.zeros((80, 128), dtype=dtype), [32, 38], CPU) == code  # spare rows are fine
    assert _check_queries(torch.zeros((1, 128), dtype=dtype), [0], CPU) == code  # a query without tokens


@pytest.mark.parametrize("q,lens", [
    (torch.zeros((70, 128), dtype=torch.float16), [70]),          # read as float32 it would be twice its size
    (torch.zeros((70, 128), dtype=torch.float64), [70]),
    (torch.zeros((70, 128), dtype=torch.int32), [70]),
    (torch.zeros((128, 70)).t(), [70]),                           # non-contiguous
    (torch.zeros((70, 64)), [70]),                                # wrong width
    (torch.zeros((70 * 128,)), [70]),                             # flat
    (torch.zeros((2, 70, 128)), [70]),
    (torch.zeros((69, 128)), [32, 38]),                           # sum(q_lens) beyond the rows
    (torch.zeros((70, 128), device=META), [70]),                  # another device
])
def test_queries_refused(q, lens):
    with pytest.raises(ValueError):
        _check_queries(q, lens, CPU)


# ------------------------------------------------------------------ device allow masks
def test_device_masks_valid():
    assert _check_device_masks(None, None, 3, 70, CPU) == (None, 0, None)
    for dt in (torch.int32, torch.uint32):
        row = torch.zeros(3, dtype=dt)
        m, n, i = _check_device_masks(row, None, 5, 70, CPU)
        assert m is row and n == 1 and i is None
        mat, idx = torch.zeros((4, 3), dtype=dt), torch.zeros(5, dtype=torch.int32)
        m, n, i = _check_device_masks(mat, idx, 5, 70, CPU)
        assert m is mat and n == 4 and i is idx
    assert _check_device_masks(torch.zeros(0, dtype=torch.int32), None, 1, 0, CPU)[1] == 1  # empty corpus: 0 words


@pytest.mark.parametrize("n_pages", [1, 31, 32, 33, 64, 70, 100])
def test_device_mask_word_count(n_pages):
    words = (n_pages + 31) // 32
    _check_device_masks(torch.zeros(words, dtype=torch.int32), None, 2, n_pages, CPU)
    idx = torch.zeros(2, dtype=torch.int32)
    _check_device_masks(torch.zeros((3, words), dtype=torch.int32), idx, 2, n_pages, CPU)
    for w in (words - 1, words + 1):
        with pytest.raises(ValueError):
            _check_device_masks(torch.zeros(w, dtype=torch.int32), None, 2, n_pages, CPU)
        with pytest.raises(ValueError):
            _check_device_masks(torch.zeros((3, w), dtype=torch.int32), idx, 2, n_pages, CPU)


I32 = torch.int32


@pytest.mark.parametrize("mask,index", [
    (None, torch.zeros(5, dtype=I32)),                            # an index without masks
    (torch.zeros(3, dtype=torch.bool), None),
    (torch.zeros(3, dtype=torch.uint8), None),
    (torch.zeros(3, dtype=torch.int64), None),
    (torch.zeros((3, 2), dtype=I32)[:, 0], None),                 # non-contiguous row
    (torch.zeros((1, 3), dtype=I32), None),                       # a matrix needs an index
    (torch.zeros(3, dtype=I32, device=META), None),
    (torch.zeros(3, dtype=I32), torch.zeros(5, dtype=I32)),       # a row with an index
    (torch.zeros((2, 4, 3), dtype=I32), torch.zeros(5, dtype=I32)),
    (torch.zeros((3, 4), dtype=I32).t(), torch.zeros(5, dtype=I32)),
    (torch.zeros((2, 3), dtype=torch.bool), torch.zeros(5, dtype=I32)),
    (torch.zeros((2, 3), dtype=I32), torch.zeros(5, dtype=torch.int64)),
    (torch.zeros((2, 3), dtype=I32), torch.zeros(4, dtype=I32)),
    (torch.zeros((2, 3), dtype=I32), torch.zeros(6, dtype=I32)),
    (torch.zeros((2, 3), dtype=I32), torch.zeros((1, 5), dtype=I32)),
    (torch.zeros((2, 3), dtype=I32), torch.zeros(10, dtype=I32)[::2]),
    (torch.zeros((2, 3), dtype=I32), torch.zeros(5, dtype=I32, device=META)),
])
def test_device_masks_refused(mask, index):
    with pytest.raises(ValueError):
        _check_device_masks(mask, index, 5, 70, CPU)


# ------------------------------------------------------------------ host allow masks
def test_host_mask_to_device():
    assert _host_mask_to_device(None, 70, CPU) is None
    words = np.array([0xFFFFFFFF, 5, 0x3F], dtype=np.uint32)
    t = _host_mask_to_device(words, 70, CPU)
    assert t.dtype == torch.int32 and t.device == CPU and np.array_equal(t.numpy().view(np.uint32), words)
    assert _host_mask_to_device([1, 2, 3], 70, CPU).tolist() == [1, 2, 3]
    for bad in (words[:2], np.zeros(4, np.uint32), np.zeros((1, 3), np.uint32)):
        with pytest.raises(ValueError):
            _host_mask_to_device(bad, 70, CPU)


# ------------------------------------------------------------------ candidate lists
def test_candidates_valid():
    assert _check_candidates(torch.zeros(7, dtype=torch.int64), 3, 5, CPU, per_query=False) == (7, 5)
    assert _check_candidates(torch.zeros(7, dtype=torch.int64), 3, 50, CPU, per_query=False) == (7, 7)
    assert _check_candidates(torch.zeros((3, 7), dtype=torch.int64), 3, 9, CPU, per_query=True) == (7, 7)
    assert _check_candidates(torch.zeros((3, 0), dtype=torch.int64), 3, 9, CPU, per_query=True) == (0, 0)


@pytest.mark.parametrize("cand,per_query", [
    (torch.zeros(7, dtype=torch.int32), False),
    (torch.zeros(7, dtype=torch.float32), False),
    (torch.zeros((3, 7), dtype=torch.int64), False),              # a shared list is one row
    (torch.zeros(14, dtype=torch.int64)[::2], False),
    (torch.zeros(7, dtype=torch.int64, device=META), False),
    (torch.zeros((3, 7), dtype=torch.int32), True),
    (torch.zeros(7, dtype=torch.int64), True),                    # one list per query
    (torch.zeros((2, 7), dtype=torch.int64), True),
    (torch.zeros((3, 7, 1), dtype=torch.int64), True),
    (torch.zeros((7, 3), dtype=torch.int64).t(), True),
    (torch.zeros((3, 7), dtype=torch.int64, device=META), True),
])
def test_candidates_refused(cand, per_query):
    with pytest.raises(ValueError):
        _check_candidates(cand, 3, 5, CPU, per_query)


# ------------------------------------------------------------------ result buffers
def test_outputs_allocated():
    ts, ti, tc = _topk_outputs(3, 5, CPU)
    assert [(tuple(t.shape), t.dtype) for t in (ts, ti, tc)] == [((3, 5), torch.float32), ((3, 5), torch.int64), ((3,), torch.int32)]
    out = _topk_outputs(3, 5, CPU, per_doc=2)
    assert [(tuple(t.shape), t.dtype) for t in out] == [((3, 5, 2), torch.float32), ((3, 5, 2), torch.int64), ((3, 5), torch.int32),
                                                        ((3,), torch.int32)]
    mine = _topk_outputs(3, 5, CPU)
    assert all(a is b for a, b in zip(_topk_outputs(3, 5, CPU, mine), mine))


@pytest.mark.parametrize("change", ["k+1", "k-1", "n_q+1", "scores_f64", "ids_i32", "counts_i64", "noncontig", "short",
                                    "meta"])
def test_outputs_refused(change):
    ts, ti, tc = _topk_outputs(3, 5, CPU)
    out = {"k+1": lambda: _topk_outputs(3, 6, CPU), "k-1": lambda: _topk_outputs(3, 4, CPU),
           "n_q+1": lambda: _topk_outputs(4, 5, CPU), "scores_f64": lambda: (ts.double(), ti, tc),
           "ids_i32": lambda: (ts, ti.int(), tc), "counts_i64": lambda: (ts, ti, tc.long()),
           "noncontig": lambda: (torch.zeros((5, 3)).t(), ti, tc), "short": lambda: (ts, ti),
           "meta": lambda: _topk_outputs(3, 5, META)}[change]()
    with pytest.raises(ValueError):
        _topk_outputs(3, 5, CPU, out)


# ------------------------------------------------------------------ the allow-mask format
def naive_words(allowed):
    w = np.zeros((len(allowed) + 31) // 32, dtype=np.uint32)
    for p in np.nonzero(allowed)[0]:
        w[p >> 5] |= np.uint32(1 << (p & 31))
    return w


def test_mask_from_pages_is_mask_words():
    rng = np.random.default_rng(5)
    for n in range(101):
        allowed = rng.random(n) < 0.5
        got = MaxSimIndex.mask_from_pages(types.SimpleNamespace(n_pages=n), allowed)
        assert got.dtype == np.uint32 and np.array_equal(got, PageCatalog.mask_words(allowed))
        assert np.array_equal(got, naive_words(allowed)), n
    with pytest.raises(ValueError):
        MaxSimIndex.mask_from_pages(types.SimpleNamespace(n_pages=40), np.ones(39, dtype=bool))


def test_stack_masks():
    a, b = np.array([1, 2], np.uint32), np.array([3, 4], np.uint32)
    mat, index = PageCatalog.stack_masks([None, a, b, a.copy(), None, b])
    assert index == [-1, 0, 1, 0, -1, 1]  # identical contents share one row, in order of first use
    assert mat.dtype == np.uint32 and mat.tolist() == [[1, 2], [3, 4]]
    assert PageCatalog.stack_masks([None, None]) == (None, [-1, -1])
    assert PageCatalog.stack_masks([]) == (None, [])


# ------------------------------------------------------------------ compaction and padding
def naive_runs(ids):
    runs = []
    for p in ids:
        if runs and p == runs[-1][1] + 1:
            runs[-1][1] = p
        else:
            runs.append([p, p])
    return [tuple(r) for r in runs]


def test_runs_match_a_naive_walk():
    rng = np.random.default_rng(7)
    cases = [[], list(range(50)), [0], [49], [0, 2, 4]]
    cases += [sorted(int(x) for x in np.nonzero(rng.random(50) < p)[0]) for p in (0.1, 0.5, 0.9) for _ in range(20)]
    for keep in cases:
        assert list(_runs(keep)) == naive_runs(keep), keep


def test_padded_lens_is_the_library_rule():
    lens = list(range(2100))
    assert _padded_lens(lens).tolist() == [nat.lib.b200ms_padded_len(n) for n in lens]
    assert _padded_lens([]).shape == (0,)


# ------------------------------------------------------------------ store
def old_record_json(r):  # the hand-written writer the journal and catalog.jsonl were first written with
    return {"document_id": r.document_id, "chunk_number": r.chunk_number, "content": r.content, "metadata": r.metadata,
            "app_id": r.app_id, "n_rows": r.n_rows}


def test_page_record_json_round_trip():
    recs = [PageRecord("d", 0, "c"), PageRecord("dé€", 7, "text \"q\"\n", {"a": [1, 2.5, None], "b": {"c": True}}, "app", 33),
            PageRecord("", -1, "", {"x": (1, 2)}, None, 0)]
    for r in recs:
        line = json.dumps(dataclasses.asdict(r))
        assert line == json.dumps(old_record_json(r))
        back = PageRecord(**json.loads(line))
        assert json.dumps(dataclasses.asdict(back)) == line


def test_capped_k(caplog):
    with caplog.at_level(logging.WARNING):
        assert _capped_k(4096) == 4096 and not caplog.records
        assert _capped_k(5000) == 4096 and "5000" in caplog.text
