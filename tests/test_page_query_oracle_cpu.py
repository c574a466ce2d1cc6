"""CPU checks of tests/page_query_oracle.py, the reference of the page-query GPU suites (test_gpu_page_query_values.py,
test_gpu_page_query_scale.py).

* From packed bytes, its page-to-page scores equal mmr_oracle.page_sum (the MMR oracle's S of two quantised pages) over the
  source's length on every dtype: exactly for int8 and 1-bit, within 1e-12 relative for bf16 and fp8.
* The comparisons those suites make reject a result that counted a tail row of the source's last group, a source read one
  page off, and examples fused in reverse order or with a fused multiply-add.
"""
import numpy as np
import pytest
import torch

import page_query_oracle as pqo
import scale_reference as sr
from explain_oracle import quantise
from mmr_oracle import page_sum
from oracle.scoring import assert_scores
from test_scale_reference_cpu import pack_pages

DTYPES = ["bf16", "int8", "fp8", "binary"]
KIND = {"bf16": "bf16", "int8": "int8", "fp8": "fp8", "binary": "bits"}
LENS = [0, 1, 31, 32, 33, 40, 65, 3]
SRC = [1, 2, 4, 6, 7, 0]


def corpus(dtype, seed=3):
    rng = np.random.default_rng(seed)
    pages = [(rng.standard_normal((n, 128)) / np.sqrt(128)).astype(np.float32) for n in LENS]
    if dtype == "int8":  # int8 codes use the whole range
        pages = [np.clip(p * 8.0, -1.0, 1.0).astype(np.float32) for p in pages]
    return pages, pack_pages(dtype, pages)


@pytest.mark.parametrize("dtype", DTYPES)
def test_reference_is_page_sum_over_length(dtype):
    pages, rows = corpus(dtype)
    got = pqo.page_query_reference(dtype, rows, LENS, SRC)
    kind = KIND[dtype]
    q = [quantise(p, kind) for p in pages]
    div = sr._score_divisor(dtype)
    want = np.array([[float(page_sum(q[s], q[j], kind)) / div / LENS[s] if LENS[s] else 0.0 for j in range(len(LENS))]
                     for s in SRC])
    if dtype in ("int8", "binary"):
        assert np.array_equal(got, want)
    else:
        np.testing.assert_allclose(got, want, rtol=1e-12, atol=0)
    assert np.all(got[SRC.index(0)] == 0.0)  # a source without rows


def test_src_block_zeroes_the_tail_and_copies_true_rows():
    pages, rows = corpus("int8")
    block, goff, q_lens = pqo.src_block(rows, LENS, SRC)
    start = pqo.starts_of(LENS)
    for i, p in enumerate(SRC):
        g0, n = 32 * int(goff[i]), LENS[p]
        assert torch.equal(block[g0:g0 + n], rows[start[p]:start[p] + n])
        assert not block[g0 + n:32 * int(goff[i + 1])].any()


@pytest.mark.parametrize("dtype", DTYPES)
def test_comparison_rejects_a_tail_row_counted(dtype):
    """A packer that left the corpus's pad rows (the page's last row repeated) in the tail of the source's last group, and a
    scan that counted them as tokens."""
    pages, rows = corpus(dtype)
    src = [1, 2, 4]  # 1, 31 and 33 rows: a tail in every last group
    want = pqo.page_query_reference(dtype, rows, LENS, src)
    start = pqo.starts_of(LENS)
    padded = [int(sr.padded_rows([LENS[p]])[0]) for p in src]
    goff = np.concatenate([[0], np.cumsum([n // 32 for n in padded])])
    block = torch.cat([rows[start[p]:start[p] + n] for p, n in zip(src, padded)])
    bad = sr.reference_from_bytes(dtype, rows, LENS, block, goff, padded).numpy() / np.asarray([LENS[p] for p in src])[:, None]
    for i in range(len(src)):
        with pytest.raises(AssertionError):
            assert_scores(dtype, bad[i], want[i], f"{dtype} tail row")


@pytest.mark.parametrize("dtype", DTYPES)
def test_comparison_rejects_a_source_one_page_off(dtype):
    pages, rows = corpus(dtype)
    src = [2, 4, 5]
    want = pqo.page_query_reference(dtype, rows, LENS, src)
    moved = pqo.page_query_reference(dtype, rows, LENS, [p + 1 for p in src])
    for i in range(len(src)):
        with pytest.raises(AssertionError):
            assert_scores(dtype, moved[i], want[i], f"{dtype} source one page off")


def test_fusion_order_and_fma_change_bits():
    rng = np.random.default_rng(9)
    s = (rng.standard_normal((4, 4096)) * 3).astype(np.float32)
    w = np.float32([0.7, -0.3, 1.1, -0.9])
    want = pqo.fuse(s, w)
    rev = pqo.fuse(s[::-1], w[::-1])
    acc = np.zeros(4096, np.float64)
    fma = np.zeros(4096, np.float32)
    for e in range(4):  # one rounding per step: acc + w * s in float64 (exact product), then to float32
        acc = fma.astype(np.float64) + np.float64(w[e]) * s[e].astype(np.float64)
        fma = acc.astype(np.float32)
    bits = lambda x: np.ascontiguousarray(x, np.float32).view(np.uint32)  # noqa: E731
    assert not np.array_equal(bits(rev), bits(want))
    assert not np.array_equal(bits(fma), bits(want))
    # the in-order fusion is numpy's own float32 arithmetic, step by step
    step = np.float32(0)
    for e in range(4):
        step = np.float32(step + np.float32(w[e] * s[e, 17]))
    assert bits(step) == bits(want[17])
