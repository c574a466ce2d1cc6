"""CPU checks of tests/scale_reference.py, the float64 MaxSim reference and corpus builder of tests/test_gpu_scale.py.

* reference_from_bytes on CPU tensors equals oracle.scoring.oracle_scores on planted corpora packed the way b200ms_pack_pages
  packs them (pages padded to 32 rows by repeating the last true row, the oracle's own quantisers): exactly for int8 and 1-bit,
  and within 1e-12 relative of a float64 numpy MaxSim for bf16 and fp8 (the C oracle itself returns float32);
* its e4m3 table and bit decoder agree with the oracle's;
* compared with assert_scores it rejects a page boundary moved by one row, a designated row deleted and two pages swapped;
* the builder's planted rows hold their margin, and its page lengths give the GPU corpora more than 1 GiB of rows past 4 GiB.
"""
import numpy as np
import pytest
import torch

import scale_reference as sr
import sign_oracle as so
from oracle import maxsim_oracle as orc
from oracle import planted
from oracle.scoring import assert_scores, oracle_scores, reference_values

DTYPES = ["bf16", "int8", "fp8", "binary"]


def pack_rows(dtype, x):
    """float32 [n, 128] -> uint8 [n, row_bytes] with the oracle's quantisers."""
    x = np.asarray(x, dtype=np.float32).reshape(-1, 128)
    if dtype == "bf16":
        return (orc.bf16_round_np(x).view(np.uint32) >> 16).astype(np.uint16).view(np.uint8).reshape(len(x), 256)
    if dtype == "int8":
        return orc.quantize_int8_np(x, 127.0).view(np.uint8)
    if dtype == "fp8":
        return orc.quantize_e4m3_np(x, 64.0)
    return orc.sign_pack_c(x).reshape(len(x), 16)


def pack_pages(dtype, pages):
    """The b200ms_pack_pages layout: every page padded to whole 32-row chunks by repeating its last true row."""
    out = []
    for p in pages:
        if len(p):
            pad = (len(p) + 31) // 32 * 32 - len(p)
            out.append(pack_rows(dtype, np.concatenate([p, np.repeat(p[-1:], pad, axis=0)])))
    return torch.from_numpy(np.concatenate(out) if out else np.zeros((0, sr.ROW_BYTES[dtype]), np.uint8))


def pack_queries(dtype, qs):
    """The packed query block: query q's tokens from row 32 * group_offsets[q], zero rows up to its last group."""
    goff = np.concatenate([[0], np.cumsum([(len(q) + 31) // 32 for q in qs])]).astype(np.int32)
    block = np.zeros((32 * int(goff[-1]), 128), np.float32)
    for q, x in zip(goff[:-1], qs):
        block[32 * q:32 * q + len(x)] = x
    return torch.from_numpy(pack_rows(dtype, block)), goff


def cpu_reference(dtype, qs, pages, **kw):
    q_u8, goff = pack_queries(dtype, qs)
    return sr.reference_from_bytes(dtype, pack_pages(dtype, pages), [len(p) for p in pages], q_u8, goff,
                                   [len(q) for q in qs], **kw).numpy()


def float64_maxsim(dtype, qs, pages):
    out = np.zeros((len(qs), len(pages)))
    for i, q in enumerate(qs):
        qv = reference_values(dtype, q)
        for p, x in enumerate(pages):
            if len(x):
                out[i, p] = (qv @ reference_values(dtype, x).T).max(axis=1).sum()
    return out


@pytest.mark.parametrize("dtype", DTYPES)
def test_reference_equals_the_oracle_on_planted_corpora(dtype):
    pc = planted.planted_corpus(dtype, seed=31, n_random=30)
    qs = planted.planted_queries(pc, [1, 32, 33, 130, 7], seed=4)
    qs.append((np.random.default_rng(2).standard_normal((45, 128)) / 11).astype(np.float32))  # mixed signs, not planted
    got = cpu_reference(dtype, qs, pc.pages)
    assert got.shape == (len(qs), len(pc.pages)) and (got[:, [p for p, n in enumerate(pc.lens) if n == 0]] == 0).all()
    want = oracle_scores(dtype, qs, pc.pages)
    if dtype in ("int8", "binary"):
        assert np.array_equal(got, want)
    else:
        f64 = float64_maxsim(dtype, qs, pc.pages)
        assert np.abs(got - f64).max() <= 1e-12 * np.abs(f64).max()
        assert np.abs(got - want).max() <= 1e-6 * np.abs(want).max()  # the C oracle's float32 output
    # a small step budget splits the corpus into many steps: the same numbers
    assert np.array_equal(cpu_reference(dtype, qs, pc.pages, budget=1), got)


def test_e4m3_table_and_bit_decoder_match_the_oracle():
    table = sr.e4m3_table().numpy()
    codes = np.arange(256, dtype=np.uint8)
    finite = (codes & 0x7F) != 0x7F
    assert np.array_equal(table[finite], orc.dequantize_e4m3_np(codes[finite]).astype(np.float64))
    assert np.isnan(table[~finite]).all()
    x = np.random.default_rng(0).standard_normal((300, 128)).astype(np.float32)
    x[0, :5] = [0.0, -0.0, 1e-30, -1e-30, np.inf]
    bits = sr.unpack_bits(torch.from_numpy(orc.sign_pack_c(x))).numpy()
    assert np.array_equal(bits, (x > 0).astype(np.uint8))
    assert np.array_equal(sr.decode("binary", torch.from_numpy(orc.sign_pack_c(x))).numpy(), np.where(x > 0, 1.0, -1.0))


@pytest.mark.parametrize("dtype", DTYPES)
def test_assert_scores_against_the_reference_rejects_layout_mutations(dtype):
    pc = planted.planted_corpus(dtype, seed=12, n_random=8)
    # one direction alone: strong on one neighbour and weak on the other, so a swap shows also where all D directions tie
    qs = [pc.directions.copy(), pc.directions[:1].copy(), *planted.planted_queries(pc, [40], seed=3)]
    pages = pc.pages
    want = cpu_reference(dtype, qs, pages)
    assert_scores(dtype, cpu_reference(dtype, qs, pages), want, "unchanged")
    p = next(i for i in range(len(pages) - 1) if len(pages[i]) > 40 and len(pages[i + 1]) > 40)
    moved = list(pages)
    moved[p], moved[p + 1] = pages[p][:-1], np.concatenate([pages[p][-1:], pages[p + 1]])
    r, _ = pc.designated[p][0]
    deleted = list(pages)
    deleted[p] = np.delete(pages[p], r, axis=0)
    swapped = list(pages)
    swapped[p], swapped[p + 1] = pages[p + 1], pages[p]
    for what, mutated in (("boundary moved by one row", moved), ("designated row deleted", deleted),
                          ("neighbouring pages swapped", swapped)):
        with pytest.raises(AssertionError):
            assert_scores(dtype, cpu_reference(dtype, qs, mutated), want, what)


@pytest.mark.parametrize("dtype", DTYPES)
def test_builder_rows_hold_their_margin(dtype):
    n_pages = 1000  # edge lengths at pages 30, 91, ... and the run of empty pages 993 .. 996
    pages, designated = [], {}
    for p0, ln, rows, pos, dir_of in sr.generate_chunks(dtype, n_pages, seed=5, device="cpu"):
        off = np.concatenate([[0], np.cumsum(ln)])
        x = rows.numpy()
        for i, n in enumerate(ln):
            pages.append(x[off[i]:off[i + 1]])
            designated[p0 + i] = [(int(r), int(d)) for r, d in zip(pos[i], dir_of[i]) if r >= 0]
    lens = np.asarray([len(p) for p in pages])
    assert (lens[993:997] == 0).all() and {1, 31, 32, 33, 127, 128, 129} <= set(lens.tolist()) and lens.max() > 1056
    assert all(len(designated[p]) == min(n, sr.D) for p, n in enumerate(lens))
    pc = planted.PlantedCorpus(dtype, pages, sr.directions(dtype, 6)[0], designated)
    planted.check_margins(pc)
    # the designated rows sweep the page, chunk and tile boundaries
    starts = np.concatenate([[0], np.cumsum(sr.padded_rows(lens))])
    cols = [int(starts[p]) + r for p, marks in designated.items() for r, _ in marks]
    assert {c % 32 for c in cols} >= {0, 31} and {c % 128 for c in cols} >= {0, 127}
    assert all(any(r == len(pages[p]) - 1 for r, _ in m) and any(r == 0 for r, _ in m) for p, m in designated.items() if m)
    # the reference of the built corpus scores every designated row: a query of one direction scores its designated row
    qs = sr.queries(dtype, 5, [8, 33])
    got = cpu_reference(dtype, qs[:1], pages[:64])
    assert_scores(dtype, got, oracle_scores(dtype, qs[:1], pages[:64]))


@pytest.mark.parametrize("dtype,n_pages", [("bf16", 20480), ("int8", 40960), ("fp8", 40960), ("binary", 327680)])
def test_gpu_corpora_reach_past_four_gib(dtype, n_pages):
    rows = int(sr.padded_rows(sr.page_lens(n_pages, 0)).sum())
    assert rows * sr.ROW_BYTES[dtype] > 2 ** 32 + 2 ** 30
    assert rows < 2 ** 31  # TMA row coordinates are int32


@pytest.mark.parametrize("dtype", ["bf16", "int8", "fp8"])
def test_sign_reference_equals_the_sign_oracle(dtype):
    # every packed value through the torch sign rule
    if dtype == "bf16":
        every = np.arange(65536, dtype=np.uint16).view(np.uint8).reshape(-1, 256)
    else:
        every = np.tile(np.arange(256, dtype=np.uint8), 64).reshape(-1, 128)
    got = sr.sign_rows_of(dtype, torch.from_numpy(every), step=7).numpy()
    assert np.array_equal(got, so.pack_bits(so.sign_bits(dtype, every)))
    # S of planted pages, and of queries without tokens and pages without rows
    pc = planted.planted_corpus(dtype, seed=33, n_random=12)
    rows = pack_pages(dtype, pc.pages)
    signs = sr.sign_rows_of(dtype, rows)
    qs = planted.planted_queries(pc, [1, 33, 0, 130], seed=5)
    q8s = [so.quantise_query(q, 127.0) for q in qs]
    want = so.scores(q8s, so.sign_bits(dtype, rows.numpy()), pc.lens)
    assert np.array_equal(sr.sign_reference(signs, pc.lens, q8s), want)
    assert np.array_equal(sr.sign_reference(signs, pc.lens, q8s, budget=1), want)
