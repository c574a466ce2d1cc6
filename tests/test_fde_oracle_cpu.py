"""The C FDE oracle (oracle/fde_oracle.c, fp32 in the device kernel's loop order) against the independent float64 numpy
restatement (oracle.maxsim_oracle.fde_encode_np), over the configuration table the GPU encoder is checked on
(tests/test_gpu_fde_matrix.py).  No GPU needed.

Rows are drawn so that every SimHash dot lies at least 1e-3 away from zero: otherwise fp32 and float64 may put a row into
different partitions, and the comparison would say nothing."""
import numpy as np
import pytest

from morphik_core_b200 import fde
from oracle import maxsim_oracle as orc

# (ksim, proj, reps, fill_empty_partitions, final_projection_dimension) -- the same table as tests/test_gpu_fde_matrix.py
CONFIGS = [
    (1, 8, 1, False, 0),      # 2 partitions, 16 of 512 threads busy
    (3, 64, 7, True, 0),      # proj 64: proj << ksim = 512
    (8, 2, 1, True, 1000),    # 256 partitions: proj << ksim = 512; final projection wider than the encoding
    (5, 16, 40, False, 0),    # the reference's partitions and projection, 40 repetitions (20480 dims)
    (8, 1, 3, False, 0),      # proj 1
    (3, 3, 7, True, 16008),   # proj 3; final projection a multiple of 8 but not of 64
    (5, 16, 20, True, 16008),
    (4, 1, 40, True, 0),
]
ITEM_ROWS = (1, 0, 2, 2047, 2048, 2049, 4097)
MARGIN = 1e-3


def cfg_of(ksim, proj, reps, fill, final):
    return fde.FixedDimensionalEncodingConfig(num_repetitions=reps, num_simhash_projections=ksim, projection_dimension=proj,
                                              fill_empty_partitions=fill, final_projection_dimension=final)


def rows_with_margin(rng, n, simhash):
    """n unit rows whose SimHash dots with every repetition's projections are all at least MARGIN away from zero."""
    G = simhash.astype(np.float64).transpose(1, 0, 2).reshape(simhash.shape[1], -1)  # [128, reps * ksim]
    x = np.zeros((n, 128), dtype=np.float32)
    todo = np.arange(n)
    while todo.size:
        y = rng.standard_normal((todo.size, 128)).astype(np.float32)
        y /= np.linalg.norm(y, axis=1, keepdims=True)
        x[todo] = y
        ok = np.abs(y.astype(np.float64) @ G).min(axis=1) >= MARGIN
        todo = todo[~ok]
    return x


def test_margin_rows_are_needed():
    """Control: without the margin, some fp32/float64 dot of a few thousand rows does land within 1e-3 of zero."""
    m = fde.fde_matrices_full(cfg_of(5, 16, 40, False, 0))
    x = np.random.default_rng(0).standard_normal((4097, 128))
    x /= np.linalg.norm(x, axis=1, keepdims=True)
    G = m.simhash.astype(np.float64).transpose(1, 0, 2).reshape(128, -1)
    assert (np.abs(x @ G) < MARGIN).any()
    assert (np.abs(rows_with_margin(np.random.default_rng(0), 4097, m.simhash).astype(np.float64) @ G) >= MARGIN).all()


@pytest.mark.parametrize("conf", CONFIGS, ids=[f"k{c[0]}-p{c[1]}-r{c[2]}-f{int(c[3])}-d{c[4]}" for c in CONFIGS])
def test_c_oracle_matches_float64_restatement(conf):
    cfg = cfg_of(*conf)
    m = fde.fde_matrices_full(cfg)
    rng = np.random.default_rng(sum(conf[:3]) + 17 * conf[4])
    proj, fill, final = cfg.projection_dimension, cfg.fill_empty_partitions, cfg.final_projection_dimension
    for n in ITEM_ROWS:
        x = rows_with_margin(rng, n, m.simhash)
        for is_doc in (False, True):
            got = orc.fde_encode_c_ex(x, m.simhash, m.ams_index, m.ams_sign, cfg.scale, is_doc, proj, fill, m.final_index,
                                      m.final_sign, final)
            want = orc.fde_encode_np(x, m.simhash, m.ams_index, m.ams_sign, cfg.scale, is_doc, proj, fill, m.final_index,
                                     m.final_sign, final)
            assert got.shape == want.shape == (cfg.fde_dimension,)
            if n == 0:
                assert not got.any() and not want.any()
                continue
            # fp32 sums of at most 4097 rows (queries) or 16 dims (sketch buckets): far inside 2e-5 of the largest entry,
            # while a row in the wrong partition, a dropped row or a wrong divisor moves some entry by more than 1e-3
            np.testing.assert_allclose(got, want, rtol=2e-5, atol=2e-5 * np.abs(want).max(), err_msg=f"{conf} n={n} doc={is_doc}")
        if fill and n in (1, 2) and not final:
            # a one- or two-point document leaves partitions empty; with fill_empty_partitions none of them stays zero
            d = orc.fde_encode_c_ex(x, m.simhash, m.ams_index, m.ams_sign, cfg.scale, True, proj, True)
            assert (np.abs(d.reshape(cfg.num_repetitions, cfg.num_partitions, proj)).sum(axis=2) > 0).all()
