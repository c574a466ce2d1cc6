"""Split launches of the wgmma scan score every page bit for bit like single-CTA passes (run with -m gpu on an H100).

A full scan of at least two resident sets of query tiles (bf16 / fp8: 2 x 4, int8 / 1-bit: 2 x 8) runs as one launch in
which CTAs 2k and 2k + 1 walk the same work units with different query tiles.  With max_ctas = 1 the same call runs
as one pass per resident set.  The raw group-score matrices of b200ms_score must be equal, at tile counts on both sides of
the split boundaries, with an odd max_ctas (rounded down to a pair), and on a corpus with fewer work units than pairs.
"""
import functools

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

torch = pytest.importorskip("torch")
if not torch.cuda.is_available():  # pragma: no cover - the gpu marker normally deselects these on CPU boxes
    pytest.skip("CUDA device required", allow_module_level=True)

from morphik_core_b200.index import MaxSimIndex  # noqa: E402
from oracle import planted  # noqa: E402

# page lengths at chunk (32) and tile (128) edges, empty pages among them
EDGE_LENS = [0, 1, 31, 32, 33, 0, 127, 128, 129, 0, 255, 256, 257, 1024, 1, 0, 1030]
RESIDENT = {"bf16": 4, "fp8": 4, "int8": 8, "binary": 8}


@functools.lru_cache(maxsize=None)
def index(dtype, n_random):
    pc = planted.planted_corpus(dtype, seed=31, n_random=n_random)
    rng = np.random.default_rng(4)
    tail = [(rng.standard_normal((n, 128)) / np.sqrt(128)).astype(np.float32) for n in EDGE_LENS]
    idx = MaxSimIndex(dtype=dtype)
    idx.add_pages(pc.pages + tail)
    idx._attach()
    return pc, idx


def queries(pc, n_tiles):
    """32-token queries filling n_tiles 128-token query tiles; the last one holds a single group."""
    return planted.planted_queries(pc, [32] * (4 * (n_tiles - 1) + 1), seed=n_tiles)


def scores(idx, qs, max_ctas):
    idx.set_option("max_ctas", max_ctas)
    try:
        s = idx.score_groups(qs)[0]
        torch.cuda.synchronize()
        return s
    finally:
        idx.set_option("max_ctas", 0)


@pytest.mark.parametrize("dtype", ["bf16", "fp8", "int8", "binary"])
@pytest.mark.parametrize("extra", [-1, 0, 1, 3])
def test_split_launch_matches_single_cta_passes(dtype, extra):
    pc, idx = index(dtype, 600)
    qs = queries(pc, 2 * RESIDENT[dtype] + extra)
    want = scores(idx, qs, 1)
    assert torch.equal(scores(idx, qs, 0), want)
    assert torch.equal(scores(idx, qs, 5), want)


@pytest.mark.parametrize("dtype", ["bf16", "int8"])
def test_fewer_units_than_pairs(dtype):
    pc, idx = index(dtype, 4)
    qs = queries(pc, 2 * RESIDENT[dtype])
    assert torch.equal(scores(idx, qs, 0), scores(idx, qs, 1))
