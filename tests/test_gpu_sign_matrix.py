"""The sign candidate stage against tests/sign_oracle.py on every input value, query length and launch shape (-m gpu, H100).

Every check is exact: integer scores S (read back with score_scale 1) and the candidate order, no tolerance.  Each part runs on
bf16, int8 and fp8 corpora, in HBM and in pinned host memory.

  * the sign rule on every packed value: crafted corpora holding every bf16 pattern at eight element positions and every int8
    / e4m3 code at all 128 positions; b200ms_sign_rows bit for bit, and the scan's S over them;
  * the query quantiser on every value: a probe corpus of single-row pages (sign_oracle.probe_bits) turns the S of a one-token
    query into its q8, for every bf16 pattern as a BF16 and as an F32 source, and for rounding ties, their one-ulp neighbours,
    +-0, subnormals, FLT_MAX, +-inf and NaNs, under scales 127, 32, 512, 1, FLT_MAX and the smallest subnormal;
  * query lengths 0 .. 1030 in batches of 1, 2, 3 (a phantom tile), 4, 8, 15, 16, 17 and 37 query tiles (the split launch
    of 2 x 8 tiles, a query whose groups straddle the two CTAs of a pair, several passes), under unit_rows default / 64 / 400
    and max_ctas 0 / 1 / 3; per-query masks with and without the filtered plan; n_cand 1 / allowed / 4096; a clamp left by a
    zero_pad_compat scan;
  * one query of 4300 tokens whose two best pages score S and S - 2 above 2^25, where float32 cannot tell them apart;
  * the two-stage search over candidate lists with unused slots, id_base, and the document search's candidate count.
"""
import ctypes

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

torch = pytest.importorskip("torch")
if not torch.cuda.is_available():  # pragma: no cover - the gpu marker normally deselects these on CPU boxes
    pytest.skip("CUDA device required", allow_module_level=True)

import sign_oracle as so  # noqa: E402
from morphik_core_b200 import _native as nat  # noqa: E402
from morphik_core_b200.index import _aligned_bytes  # noqa: E402
from morphik_core_b200.signs import SignTwoStageIndex  # noqa: E402
from oracle.planted import planted_corpus, planted_queries  # noqa: E402

DEV = torch.device("cuda", 0)
DTYPES = ("bf16", "int8", "fp8")
TIERS = ("hbm", "host")
CORPORA = [(d, t) for d in DTYPES for t in TIERS]
Q_SCALE = 127.0
FLT_MAX = float(np.finfo(np.float32).max)
FLT_TRUE_MIN = float(np.float32(2.0 ** -149))
SCALES = (127.0, 32.0, 512.0, 1.0, FLT_MAX, FLT_TRUE_MIN)
DEFAULT_UNIT_ROWS = 4096
# the planted corpus, repeated: about 265 000 rows, so that a 400-row unit cap binds (set_corpus sizes units to
# rows / (4 * SMs), at least 128 rows, at most unit_rows) and the default plan has several hundred units
REPEATS = 16


def cstream():
    return ctypes.c_void_p(torch.cuda.current_stream(DEV).cuda_stream)


def sign_call(sti, src, lens, n_cand, scale=Q_SCALE, masks=None, index=None):
    """b200ms_sign_candidates_device on device rows src (float32 | bfloat16) with score_scale 1: scores are float32(S)."""
    n_q = len(lens)
    ts = torch.empty((n_q, n_cand), dtype=torch.float32, device=DEV)
    ti = torch.empty((n_q, n_cand), dtype=torch.int64, device=DEV)
    tc = torch.empty((n_q,), dtype=torch.int32, device=DEV)
    sti._attach()
    rc = nat.lib.b200ms_sign_candidates_device(
        sti.index.h.ptr, ctypes.c_void_p(src.data_ptr()), nat.BF16 if src.dtype == torch.bfloat16 else nat.F32,
        nat.i32_array(lens), n_q, n_cand, None if masks is None else ctypes.c_void_p(masks.data_ptr()),
        0 if masks is None else masks.shape[0], None if index is None else ctypes.c_void_p(index.data_ptr()),
        ctypes.c_float(scale), ctypes.c_float(1.0), ctypes.c_void_p(ts.data_ptr()), ctypes.c_void_p(ti.data_ptr()),
        ctypes.c_void_p(tc.data_ptr()), cstream())
    sti.index.h.check(rc, "b200ms_sign_candidates_device")
    return ts.cpu().numpy(), ti.cpu().numpy(), tc.cpu().numpy()


def stage(queries):
    """Host float32 queries -> one device float32 tensor (at least one row) and their lengths."""
    lens = [int(q.shape[0]) for q in queries]
    rows = np.concatenate([np.asarray(q, np.float32).reshape(-1, 128) for q in queries] + [np.zeros((0, 128), np.float32)])
    if len(rows) == 0:
        rows = np.zeros((1, 128), np.float32)
    return torch.from_numpy(np.ascontiguousarray(rows)).to(DEV), lens


def check(res, S, n_cand, allowed=None, what=""):
    """Candidates = sign_oracle.topk of the exact S among each query's allowed pages; scores float32(S) bit for bit."""
    ts, ti, tc = res
    for q in range(S.shape[0]):
        want = so.topk(S[q], n_cand, None if allowed is None else allowed[q])
        assert tc[q] == len(want), (what, q)
        assert ti[q, :len(want)].tolist() == want, (what, q)
        assert np.array_equal(ts[q, :len(want)].view(np.uint32), S[q, want].astype(np.float32).view(np.uint32)), (what, q)
        assert (ti[q, len(want):] == -1).all() and np.isneginf(ts[q, len(want):]).all(), (what, q)


def all_scores(res, n_pages):
    """S [n_q, n_pages] of a call whose n_cand covers every page."""
    ts, ti, tc = res
    S = np.full((len(tc), n_pages), np.nan)
    for q in range(len(tc)):
        assert tc[q] == n_pages
        S[q, ti[q, :n_pages]] = ts[q, :n_pages]
    assert not np.isnan(S).any()
    return S.astype(np.int64)


def sign_index(dtype, tier, pages=None, packed=None, n_pages=0):
    sti = SignTwoStageIndex(dtype=dtype, tier=tier, q_scale=Q_SCALE)
    if pages is not None:
        sti.add_pages(pages)
    else:
        buf = _aligned_bytes(packed.nbytes, DEV)
        buf.copy_(torch.from_numpy(packed.reshape(-1)))
        sti.adopt_packed(buf, [32] * n_pages)
    torch.cuda.synchronize(DEV)
    return sti


def corpus_bits(dtype, sti):
    return so.sign_bits(dtype, sti.index.packed_rows().cpu().numpy())


# ------------------------------------------------------------------------------------------------ 1. the sign rule
def crafted_rows(dtype):
    """Packed rows, 32 per page: bf16 -- every pattern at 8 element positions (row block s rotates by 37 s); int8 / fp8 --
    code (r + i) mod 256 at element i of row r, every code at every position."""
    if dtype == "bf16":
        v = np.arange(65536, dtype=np.int64).reshape(512, 128)
        blocks = [np.roll(v, -37 * s, axis=1) for s in range(8)]
        return np.concatenate(blocks).astype("<u2").view(np.uint8).reshape(-1, 256)
    r, i = np.meshgrid(np.arange(256), np.arange(128), indexing="ij")
    return ((r + i) % 256).astype(np.uint8)


@pytest.mark.parametrize("dtype,tier", CORPORA)
def test_sign_rule_on_every_packed_value(dtype, tier):
    packed = crafted_rows(dtype)
    n_pages = len(packed) // 32
    sti = sign_index(dtype, tier, packed=packed, n_pages=n_pages)
    try:
        bits = so.sign_bits(dtype, packed)
        np.testing.assert_array_equal(sti.sign_rows().cpu().numpy(), so.pack_bits(bits))
        rng = np.random.default_rng(5)
        qs = [(rng.standard_normal((t, 128)) * rng.choice([0.05, 0.3, 1.0], size=(t, 1))).astype(np.float32)
              for t in (1, 40, 7)]
        src, lens = stage(qs)
        S = so.scores([so.quantise_query(q, Q_SCALE) for q in qs], bits, [32] * n_pages)
        check(sign_call(sti, src, lens, n_pages), S, n_pages, what=f"{dtype} {tier}")
    finally:
        sti.index.close()


# ------------------------------------------------------------------------------------------------ 2. the quantiser
def probe_pages():
    """The probe corpus as float pages: page 0 all -1, page 1 + i all -1 but +1 at element i (every dtype keeps the signs)."""
    pages = [-np.ones((1, 128), np.float32)]
    for i in range(128):
        p = -np.ones((1, 128), np.float32)
        p[0, i] = 1.0
        pages.append(p)
    return pages


def special_f32():
    """float32 bit patterns the quantiser singles out: +-0, the smallest and largest subnormals, FLT_MAX, +-inf, quiet,
    signalling and negative NaNs."""
    bits = [0x00000000, 0x80000000, 0x00000001, 0x80000001, 0x007FFFFF, 0x807FFFFF, 0x7F7FFFFF, 0xFF7FFFFF,
            0x7F800000, 0xFF800000, 0x7FC00000, 0xFFC00000, 0x7F800001, 0xFF800001, 0x7FBFFFFF, 0x7FFFFFFF, 0xFFFFFFFF]
    return np.array(bits, dtype=np.uint32).view(np.float32)


def targeted_f32(scale):
    ties = so.tie_inputs(scale)
    up = np.nextafter(ties, np.float32(np.inf), dtype=np.float32)
    down = np.nextafter(ties, np.float32(-np.inf), dtype=np.float32)
    return np.concatenate([ties, up, down, special_f32()])


def one_token_queries(values):
    """float32 values -> [n, 128] rows (zero padded): one one-token query per row."""
    n = (len(values) + 127) // 128
    x = np.zeros(n * 128, dtype=np.float32)
    x[:len(values)] = values
    return x.reshape(n, 128)


@pytest.fixture(scope="module", params=CORPORA, ids=lambda p: f"{p[0]}-{p[1]}")
def probe(request):
    dtype, tier = request.param
    sti = sign_index(dtype, tier, pages=probe_pages())
    np.testing.assert_array_equal(corpus_bits(dtype, sti)[::32], so.probe_bits())
    yield sti
    torch.cuda.synchronize(DEV)
    sti.index.close()


def probe_q8(sti, src, n_q, scale):
    return so.probe_q8(all_scores(sign_call(sti, src, [1] * n_q, 129, scale=scale), 129))


@pytest.mark.parametrize("scale", SCALES, ids=lambda s: f"{s:g}")
def test_quantiser_on_every_bf16_value(probe, scale):
    u16 = np.arange(65536, dtype=np.uint32)
    wide = (u16 << 16).view(np.float32).reshape(512, 128)  # exact widening: NaN payloads and signalling NaNs kept
    want = so.quantise_query(wide, scale)
    bf = torch.from_numpy(u16.astype(np.uint16).view(np.int16).reshape(512, 128)).view(torch.bfloat16).to(DEV)
    np.testing.assert_array_equal(probe_q8(probe, bf, 512, scale), want, err_msg="BF16 source")
    np.testing.assert_array_equal(probe_q8(probe, torch.from_numpy(wide).to(DEV), 512, scale), want, err_msg="F32 source")


@pytest.mark.parametrize("scale", SCALES, ids=lambda s: f"{s:g}")
def test_quantiser_on_ties_and_special_values(probe, scale):
    x = targeted_f32(scale)
    q = one_token_queries(x)
    got = probe_q8(probe, torch.from_numpy(q).to(DEV), len(q), scale).reshape(-1)[:len(x)]
    np.testing.assert_array_equal(got, so.quantise_query(q, scale).reshape(-1)[:len(x)])
    if scale in (32.0, 512.0, 1.0):  # every k + 0.5 is reachable: both rounding directions and both clamps are exercised
        ties = got[:128]
        assert (ties % 2 == 0).sum() == 128 - 2 and set(ties[[0, -1]].tolist()) == {-63, 63}


# ------------------------------------------------------------------------------------------------ 3. lengths and launches
def groups(lens):
    return sum((t + 31) // 32 for t in lens)


def tiles(lens):
    return (groups(lens) + 3) // 4 * 4 // 4


# batches named by their query tiles (4 groups of 32 tokens each); "16" puts a 1030-token query on groups 30 .. 62, across
# the two halves (8 tiles each) of the split launch
BATCHES = {
    "1": [0, 1, 31, 64],
    "2": [127, 128, 0],
    "3 (phantom)": [300],
    "4": [300, 33, 64],
    "8": [300, 300, 129, 127],
    "15": [1030, 300, 127, 64, 31, 128, 129],
    "16": [300, 300, 300, 1030],
    "17": [300, 300, 300, 1030, 64],
    "37 (passes)": [1030, 1030, 1030, 1030, 300, 129, 1],
}
LAUNCHES = [(u, m) for u in (DEFAULT_UNIT_ROWS, 64, 400) for m in (0, 1, 3)]
_oracle_cache = {}


@pytest.fixture(scope="module", params=CORPORA, ids=lambda p: f"{p[0]}-{p[1]}")
def planted(request):
    dtype, tier = request.param
    pc = planted_corpus(dtype, seed=3)
    sti = sign_index(dtype, tier, pages=pc.pages * REPEATS)
    base_bits = so.sign_bits(dtype, sti.index.packed_rows()[:int(so.page_starts(pc.lens)[-1])].cpu().numpy())
    yield dtype, pc, sti, base_bits
    torch.cuda.synchronize(DEV)
    sti.index.close()


def batch_oracle(dtype, pc, base_bits, name, seed):
    """Queries of batch `name` and their S over the repeated corpus (the S of the planted pages, repeated)."""
    key = (dtype, name, seed)
    if key not in _oracle_cache:
        qs = planted_queries(pc, BATCHES[name], seed=seed)
        S = so.scores([so.quantise_query(q, Q_SCALE) for q in qs], base_bits, pc.lens)
        _oracle_cache[key] = (qs, np.tile(S, REPEATS))
    return _oracle_cache[key]


def set_launch(sti, unit_rows, max_ctas):
    sti.index.set_option("unit_rows", unit_rows)  # detaches: the next call re-attaches with the new units
    sti.index.set_option("max_ctas", max_ctas)


def test_batches_have_their_tile_counts():
    for name, lens in BATCHES.items():
        assert tiles(lens) == int(name.split()[0]), name
    assert groups([300] * 3) < 32 < groups([300] * 3 + [1030]) <= 64  # the 1030-token query straddles the split


@pytest.mark.parametrize("name", list(BATCHES))
def test_lengths_and_launch_shapes(planted, name):
    dtype, pc, sti, base_bits = planted
    qs, S = batch_oracle(dtype, pc, base_bits, name, seed=1)
    src, lens = stage(qs)
    try:
        for unit_rows, max_ctas in LAUNCHES:
            set_launch(sti, unit_rows, max_ctas)
            check(sign_call(sti, src, lens, 4096), S, 4096, what=f"{name} unit_rows={unit_rows} max_ctas={max_ctas}")
    finally:
        set_launch(sti, DEFAULT_UNIT_ROWS, 0)


@pytest.mark.parametrize("name", ["1", "4", "16", "37 (passes)"])
def test_masks_with_and_without_the_filtered_plan(planted, name):
    dtype, pc, sti, base_bits = planted
    qs, S = batch_oracle(dtype, pc, base_bits, name, seed=2)
    src, lens = stage(qs)
    n, n_q = sti.n_pages, len(qs)
    rng = np.random.default_rng(11)
    mats = rng.integers(0, 2 ** 32, size=(3, (n + 31) // 32), dtype=np.uint64).astype(np.uint32)
    mats[1] &= rng.integers(0, 2 ** 32, size=mats.shape[1], dtype=np.uint64).astype(np.uint32)  # about a quarter
    mats[2] = 0
    mats[2, 0] = 0b100110  # pages 1, 2, 5
    allow = [so.mask_allowed(m, n) for m in mats]
    index = np.array([(-1, 0, 1, 2)[q % 4] for q in range(n_q)], dtype=np.int32)
    rows = [None if i < 0 else allow[i] for i in index]
    masks_dev = torch.from_numpy(mats.view(np.int32)).to(DEV)
    index_dev = torch.from_numpy(index).to(DEV)
    try:
        # max_ctas 0 and 8: fewer CTAs than units, the filtered plan; 4096: at least one CTA per unit, the corpus' own plan
        for max_ctas in (0, 8, 4096):
            sti.index.set_option("max_ctas", max_ctas)
            for n_cand in (1, int(max(a.sum() for a in allow)), 4096):
                check(sign_call(sti, src, lens, n_cand, masks=masks_dev, index=index_dev), S, n_cand, rows,
                      f"{name} max_ctas={max_ctas} n_cand={n_cand}")
    finally:
        sti.index.set_option("max_ctas", 0)


def test_a_scale_that_zeroes_every_q8_ties_every_page(planted):
    dtype, pc, sti, _ = planted
    qs = planted_queries(pc, [33, 1, 300], seed=4)
    qs[1] = np.full((1, 128), FLT_MAX, np.float32)  # the largest finite value still rounds to 0 under the smallest scale
    src, lens = stage(qs)
    n = sti.n_pages
    assert any(ln == 0 for ln in pc.lens)
    S = np.zeros((len(qs), n), dtype=np.int64)
    check(sign_call(sti, src, lens, 4096, scale=FLT_TRUE_MIN), S, 4096, what="zero q8")
    words = np.random.default_rng(3).integers(0, 2 ** 32, size=(1, (n + 31) // 32), dtype=np.uint64).astype(np.uint32)
    allowed = so.mask_allowed(words[0], n)
    res = sign_call(sti, src, lens, 4096, scale=FLT_TRUE_MIN, masks=torch.from_numpy(words.view(np.int32)).to(DEV),
                    index=torch.zeros(len(qs), dtype=torch.int32, device=DEV))
    check(res, S, 4096, [allowed] * len(qs), "zero q8, masked")
    assert res[1][0, :int(allowed.sum())].tolist() == np.flatnonzero(allowed).tolist()


def test_a_zero_pad_compat_clamp_stays_out_of_S(planted):
    dtype, pc, sti, base_bits = planted
    qs, S = batch_oracle(dtype, pc, base_bits, "4", seed=1)
    src, lens = stage(qs)
    idx = sti.index
    idx.set_option("zero_pad_compat", 128)
    try:
        if idx.tier == "hbm":  # a full scan with the clamp: it leaves the corpus' clamp bits on the handle
            idx.search_device(src, lens, 10)
        cand = torch.arange(0, 64, dtype=torch.int64, device=DEV).repeat(len(qs), 1).contiguous()
        idx.rerank_batch(src, lens, cand, 10)  # a rerank with the clamp: clamp bits per candidate slot
        check(sign_call(sti, src, lens, 4096), S, 4096, what="after zero_pad_compat scans")
    finally:
        idx.set_option("zero_pad_compat", 0)


# ------------------------------------------------------------------------------------------------ S past 2^25
@pytest.mark.parametrize("dtype,tier", CORPORA)
def test_exact_order_where_float32_ties(dtype, tier):
    """Two single-row pages, equal but for the sign of element j, and a 4300-token query: every token is 1 (q8 = 63) but
    element j, which is 0 except in the last token, where its q8 is 1.  S differs by 2 between the pages, above 2^25."""
    j, T = 77, 4300
    lo, hi = np.ones((1, 128), np.float32), np.ones((1, 128), np.float32)
    lo[0, j] = -1.0
    sti = sign_index(dtype, tier, pages=[lo, hi, -np.ones((1, 128), np.float32)])
    try:
        q = np.ones((T, 128), np.float32)
        q[:, j] = 0.0
        q[-1, j] = np.float32(1.0 / Q_SCALE)
        q8 = so.quantise_query(q, Q_SCALE)
        assert (np.delete(q8, j, axis=1) == 63).all() and (q8[:-1, j] == 0).all() and q8[-1, j] == 1
        S = so.scores([q8], corpus_bits(dtype, sti), [1, 1, 1])
        assert S[0, 1] - S[0, 0] == 2 and S[0, 0] > 2 ** 25 and np.float32(S[0, 0]) == np.float32(S[0, 1])
        src, lens = stage([q])
        res = sign_call(sti, src, lens, 3)
        check(res, S, 3, what=f"{dtype} {tier}")
        assert res[1][0].tolist() == [1, 0, 2]  # a float32 key would tie pages 0 and 1 and put page 0 first
    finally:
        sti.index.close()


# ------------------------------------------------------------------------------------------------ 4. the two-stage search
@pytest.mark.parametrize("dtype,tier", CORPORA)
def test_two_stage_over_lists_with_unused_slots(dtype, tier):
    pc = planted_corpus(dtype, seed=5)
    sti = sign_index(dtype, tier, pages=pc.pages)
    try:
        n = sti.n_pages
        qs = planted_queries(pc, [1, 33, 64, 130], seed=6)
        src, lens = stage(qs)
        allowed = np.zeros(n, bool)
        empty = pc.lens.index(0)
        allowed[[1, 4, empty, 40, 41, n - 1]] = True  # six pages, one without rows: fewer than k, fewer than n_candidates
        assert allowed.sum() == 6
        mask = torch.from_numpy(sti.index.mask_from_pages(allowed).view(np.int32)).to(DEV)
        for n_candidates in (50, 3):
            _, ci, _ = sti.candidates_device(src, lens, sti._n_cand(max(n_candidates, 10)), mask)
            assert (ci[:, 6:] == -1).all() and (ci[:, :6] >= 0).all()
            want = sti.index.rerank_batch(src, lens, ci, 10)
            assert (want[1][:, 6:] == -1).all()
            for id_base in (0, 1000):
                got = sti.search_device(qs, 10, n_candidates=n_candidates, allow_mask_dev=mask, id_base=id_base)[:3]
                shifted = torch.where(want[1] >= 0, want[1] + id_base, want[1])
                assert torch.equal(got[0], want[0]) and torch.equal(got[1], shifted) and torch.equal(got[2], want[2])
        # documents: k * per_doc = 12 candidates, more than n_candidates = 5
        page_doc = (torch.arange(n, dtype=torch.int32, device=DEV) // 4).contiguous()
        n_docs = (n + 3) // 4
        got = sti.search_docs_device(qs, 4, 3, page_doc, n_docs, n_candidates=5)
        _, ci, _ = sti.candidates_device(src, lens, 12)
        want = sti.index.rerank_docs_batch(src, lens, ci, 4, 3, page_doc, n_docs)
        for a, b in zip(got, want):
            assert torch.equal(a, b)
        _, c5, _ = sti.candidates_device(src, lens, 5)
        short = sti.index.rerank_docs_batch(src, lens, c5, 4, 3, page_doc, n_docs)
        assert not all(torch.equal(a, b) for a, b in zip(short, want))  # the max() is observable
    finally:
        sti.index.close()
