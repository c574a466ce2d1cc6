"""The pack kernels on every input value (run with -m gpu on an H100): b200ms_pack_pages, b200ms_pack_queries and
b200ms_sign_pack called through the C-ABI, their output BYTES compared with oracle/value_rules.py (torch integer and table
operations, tied to the numpy oracle by tests/test_value_oracle_cpu.py).

(a) every float32 bit pattern, as an F32 source, to bf16, int8 (scales 127 and 1), fp8 (scales 64 and 48) and 1-bit, and
    through b200ms_sign_pack -- exhaustively, in chunks of 2^26 patterns (256 MiB of source);
(b) every bf16 bit pattern as a BF16 source, to every dtype, as pages and as queries;
(c) the layout contract: page pad rows repeat the last true row, empty pages take no rows, query pad rows and the tail
    up to roundup(groups, 4) * 32 rows are zero, nothing past the layout is written;
(d) scores of corpora made of the special values (ties, subnormals, saturation, signed zeros) against the oracle, with
    BF16 query sources.
Every destination is pre-filled with 0xA5 so that a row the kernel leaves unwritten shows up.
"""
import ctypes

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

torch = pytest.importorskip("torch")
if not torch.cuda.is_available():  # pragma: no cover - the gpu marker normally deselects these on CPU boxes
    pytest.skip("CUDA device required", allow_module_level=True)

from morphik_core_b200 import _native as nat  # noqa: E402
from morphik_core_b200.index import MaxSimIndex  # noqa: E402
from oracle import maxsim_oracle as orc  # noqa: E402
from oracle import value_rules as vr  # noqa: E402
from oracle.scoring import assert_scores, oracle_scores  # noqa: E402

DT = {"bf16": nat.BF16, "int8": nat.I8, "fp8": nat.F8, "binary": nat.B1}
SCALE = {"bf16": 1.0, "int8": 127.0, "fp8": 64.0, "binary": 1.0}
FILL = 0xA5
CHUNK = 1 << 26  # float32 patterns per pack call: 256 MiB of source
PAGE = 32


@pytest.fixture(scope="module")
def h():
    return nat.Handle(0)


def vp(t):
    return ctypes.c_void_p(t.data_ptr())


def stream():
    return ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)


def filled(nbytes):
    return torch.full((nbytes,), FILL, dtype=torch.uint8, device="cuda")


def pack_pages(h, src, src_dtype, lens, dtype, scale, extra_rows=0):
    """b200ms_pack_pages into a 0xA5-filled buffer of padded_rows + extra_rows rows -> uint8 [rows, row_bytes]."""
    lens_c = nat.i32_array(lens)
    rows = int(nat.lib.b200ms_padded_rows(lens_c, len(lens)))
    rb = nat.ROW_BYTES[DT[dtype]]
    out = filled((rows + extra_rows) * rb)
    h.check(nat.lib.b200ms_pack_pages(h.ptr, vp(src), src_dtype, lens_c, len(lens), vp(out), DT[dtype], ctypes.c_float(scale),
                                      stream()), "b200ms_pack_pages")
    torch.cuda.synchronize()
    return out.view(-1, rb)


def pack_queries(h, src, src_dtype, lens, dtype, scale, extra_rows=0):
    lens_c = nat.i32_array(lens)
    groups = int(nat.lib.b200ms_query_groups(lens_c, len(lens)))
    cap = (groups + 3) // 4 * 4 * PAGE
    rb = nat.ROW_BYTES[DT[dtype]]
    out = filled((cap + extra_rows) * rb)
    goff = (ctypes.c_int32 * (len(lens) + 1))()
    ng = ctypes.c_int(-1)
    h.check(nat.lib.b200ms_pack_queries(h.ptr, vp(src), src_dtype, lens_c, len(lens), vp(out), DT[dtype], ctypes.c_float(scale),
                                        goff, ctypes.byref(ng), stream()), "b200ms_pack_queries")
    torch.cuda.synchronize()
    return out.view(-1, rb), list(goff), ng.value, groups, cap


def assert_bytes(got, want, bits, what):
    """got / want uint8 [rows, row_bytes] on the device; bits the [rows, 128] int32 source patterns."""
    if torch.equal(got, want):
        return
    bad = (got != want).nonzero()[:5].tolist()
    rb = got.shape[1]
    detail = []
    for r, c in bad:
        e = c * 8 if rb == 16 else (c // 2 if rb == 256 else c)
        detail.append((f"pattern 0x{int(bits[r, e]) & 0xFFFFFFFF:08x}", f"got 0x{int(got[r, c]):02x}", f"want 0x{int(want[r, c]):02x}"))
    raise AssertionError(f"{what}: {int((got != want).sum())} bytes differ, first {detail}")


# ------------------------------------------------------------------------------------------------ (a) every float32
SWEEPS = [("bf16", 1.0), ("int8", 127.0), ("int8", 1.0), ("fp8", 64.0), ("fp8", 48.0), ("binary", 1.0)]


@pytest.mark.parametrize("dtype,scale", SWEEPS, ids=[f"{d}-{s:g}" for d, s in SWEEPS])
def test_every_float32_pattern_packs_exactly(h, dtype, scale):
    lens = [PAGE] * (CHUNK // 128 // PAGE)
    base = torch.arange(CHUNK, dtype=torch.int32, device="cuda")
    for c in range((1 << 32) // CHUNK):
        bits = (base + (c * CHUNK - (1 << 31))).view(-1, 128)  # int32 adds without overflow: patterns -2^31 .. 2^31-1
        got = pack_pages(h, bits.view(torch.float32), nat.F32, lens, dtype, scale)
        assert_bytes(got, vr.packed_bytes(dtype, bits, scale), bits, f"{dtype} scale {scale} chunk {c}")


def test_every_float32_pattern_sign_packs_exactly(h):
    base = torch.arange(CHUNK, dtype=torch.int32, device="cuda")
    rows = CHUNK // 128
    for c in range((1 << 32) // CHUNK):
        bits = (base + (c * CHUNK - (1 << 31))).view(-1, 128)
        out = filled(rows * 16 + 16)
        h.check(nat.lib.b200ms_sign_pack(h.ptr, vp(bits), nat.F32, rows, vp(out), stream()), "b200ms_sign_pack")
        torch.cuda.synchronize()
        assert torch.all(out[rows * 16:] == FILL)
        assert_bytes(out[: rows * 16].view(-1, 16), vr.sign_bytes(bits), bits, f"sign_pack chunk {c}")


# ------------------------------------------------------------------------------------------------ (b) every bf16
def all_bf16():
    """Every bf16 pattern as a [512, 128] BF16 tensor, and the float32 patterns it widens to."""
    b16 = torch.arange(-(1 << 15), 1 << 15, dtype=torch.int32, device="cuda")
    src = b16.to(torch.int16).view(torch.bfloat16).view(-1, 128).contiguous()
    bits = (b16 << 16).view(-1, 128)  # the exact float32 widening: the low 16 bits are zero
    return src, bits


@pytest.mark.parametrize("dtype", list(DT))
def test_every_bf16_pattern_packs_exactly_as_pages_and_queries(h, dtype):
    src, bits = all_bf16()
    scale = SCALE[dtype]
    want = vr.packed_bytes(dtype, bits, scale)
    got = pack_pages(h, src, nat.BF16, [PAGE] * (bits.shape[0] // PAGE), dtype, scale)
    assert_bytes(got, want, bits, f"pages {dtype}")
    got_q, goff, ng, groups, cap = pack_queries(h, src, nat.BF16, [PAGE] * (bits.shape[0] // PAGE), dtype, scale)
    assert ng == groups == bits.shape[0] // PAGE and cap == bits.shape[0]  # 16 groups: no pad rows, no tail
    assert_bytes(got_q, want, bits, f"queries {dtype}")


def test_every_bf16_pattern_sign_packs_exactly(h):
    src, bits = all_bf16()
    rows = bits.shape[0]
    out = filled(rows * 16)
    h.check(nat.lib.b200ms_sign_pack(h.ptr, vp(src), nat.BF16, rows, vp(out), stream()), "b200ms_sign_pack")
    torch.cuda.synchronize()
    assert_bytes(out.view(-1, 16), vr.sign_bytes(bits), bits, "sign_pack bf16")


# ------------------------------------------------------------------------------------------------ (c) layout contract
PAGE_LENS = [1, 0, 31, 32, 33, 0, 64, 1030]
QUERY_LENS = [1, 0, 32, 33, 0, 5, 70]  # 1 + 1 + 2 + 1 + 3 = 8 groups
QUERY_LENS_TAIL = [33, 0, 1]  # 3 groups -> capacity 4 groups: one whole tail group


def random_bits(rng, n):
    """Gaussian rows with a sprinkling of special values, as float32 patterns [n, 128] on the device."""
    x = (rng.standard_normal((n, 128)) * 0.3).astype(np.float32)
    sp = np.asarray([0.0, -0.0, np.inf, -np.inf, np.nan, 1e-40, -1e-40, 7.5, -9.0], np.float32)
    m = rng.random((n, 128)) < 0.05
    x[m] = rng.choice(sp, size=int(m.sum()))
    return torch.from_numpy(x.view(np.int32)).cuda()


@pytest.mark.parametrize("src_dtype", ["f32", "bf16"])
@pytest.mark.parametrize("dtype", list(DT))
def test_page_layout_repeats_last_row_and_skips_empty_pages(h, dtype, src_dtype):
    rng = np.random.default_rng(11)
    bits = random_bits(rng, sum(PAGE_LENS))
    if src_dtype == "bf16":
        src = bits.view(torch.float32).bfloat16()
        bits = (src.view(torch.int16).to(torch.int32) << 16).contiguous()
    else:
        src = bits.view(torch.float32)
    scale = SCALE[dtype]
    got = pack_pages(h, src, nat.F32 if src_dtype == "f32" else nat.BF16, PAGE_LENS, dtype, scale, extra_rows=3)
    rows = vr.packed_bytes(dtype, bits, scale)
    parts, s = [], 0
    for n in PAGE_LENS:
        if n:
            parts.append(rows[s:s + n])
            parts.append(rows[s + n - 1:s + n].expand((-n) % PAGE, -1))  # pad rows: the last true row, byte for byte
        s += n
    want = torch.cat(parts)
    assert want.shape[0] == sum((n + PAGE - 1) // PAGE * PAGE for n in PAGE_LENS)
    assert_bytes(got[: want.shape[0]], want, _row_bits(bits, PAGE_LENS), f"pages {dtype} from {src_dtype}")
    assert torch.all(got[want.shape[0]:] == FILL)  # nothing written past the layout


def _row_bits(bits, lens):
    """Source patterns of every padded row (pad rows: the page's last true row), for mismatch reports."""
    idx, s = [], 0
    for n in lens:
        if n:
            idx += list(range(s, s + n)) + [s + n - 1] * ((-n) % PAGE)
        s += n
    return bits[torch.as_tensor(idx, device=bits.device)]


@pytest.mark.parametrize("lens", [QUERY_LENS, QUERY_LENS_TAIL], ids=["8groups", "tail"])
@pytest.mark.parametrize("dtype", list(DT))
def test_query_layout_zero_pads_and_reports_groups(h, dtype, lens):
    rng = np.random.default_rng(12)
    bits = random_bits(rng, sum(lens))
    scale = SCALE[dtype]
    got, goff, ng, groups, cap = pack_queries(h, bits.view(torch.float32), nat.F32, lens, dtype, scale, extra_rows=2)
    want_goff = np.concatenate([[0], np.cumsum([(n + PAGE - 1) // PAGE for n in lens])]).tolist()
    assert goff == want_goff and ng == groups == want_goff[-1]
    rows = vr.packed_bytes(dtype, bits, scale)
    want = torch.zeros((cap, rows.shape[1]), dtype=torch.uint8, device="cuda")  # pad rows and the tail: zero bytes
    s = 0
    for i, n in enumerate(lens):
        want[goff[i] * PAGE: goff[i] * PAGE + n] = rows[s:s + n]
        s += n
    src_rows = torch.zeros((cap, 128), dtype=torch.int32, device="cuda")
    assert_bytes(got[:cap], want, src_rows, f"queries {dtype} {lens}")
    assert torch.all(got[cap:] == FILL)  # capacity is roundup(groups, 4) * 32 rows: nothing past it


# ------------------------------------------------------------------------------------------------ (d) end to end
def special_rows(rng, n):
    """Rows drawn from finite special values: signed zeros, subnormals of both signs, the smallest normal, bf16 ties, int8
    ties at scale 127, e4m3 ties and subnormals at scale 64, int8 / e4m3 saturation.  Apart from the zeros and the
    subnormals the values are positive, so that no dot product cancels to near zero (the bf16 / fp8 bars are relative)."""
    tiny = np.asarray([1e-45, 1e-40, 1.1754944e-38], np.float32)
    ties = np.asarray([1 + 2 ** -8, 1 + 3 * 2 ** -8, 0.5 / 127, 1.5 / 127, 2.5 / 127, 126.5 / 127, 1.0625 / 64,
                       1.1875 / 64, 2 ** -10 / 64, 3 * 2 ** -10 / 64, 0.7, 0.25], np.float32)
    sat = np.asarray([1.5, 7.5, 9.0], np.float32)
    x = rng.choice(np.concatenate([ties, sat]).astype(np.float32), size=(n, 128))
    m = rng.random((n, 128)) < 0.15
    x[m] = rng.choice(np.concatenate([tiny, -tiny]).astype(np.float32), size=int(m.sum()))
    x[rng.random((n, 128)) < 0.1] = np.float32(-0.0)
    x[rng.random((n, 128)) < 0.1] = np.float32(0.0)
    return x.astype(np.float32)


@pytest.mark.parametrize("dtype", list(DT))
def test_special_value_corpus_scores_match_oracle_with_bf16_queries(dtype):
    rng = np.random.default_rng(21)
    lens = [1, 31, 32, 33, 0, 64, 5, 130] + [int(v) for v in rng.integers(1, 90, size=30)]
    pages = [special_rows(rng, n) for n in lens]
    q32 = [orc.bf16_round_np(special_rows(rng, t)) for t in (32, 7, 33, 64)]  # bf16-exact: the BF16 source holds them
    qbf = [torch.from_numpy(q).cuda().bfloat16() for q in q32]
    assert all(np.array_equal(b.float().cpu().numpy(), q) for b, q in zip(qbf, q32))
    idx = MaxSimIndex(dtype=dtype)
    idx.add_pages(pages)
    want = oracle_scores(dtype, q32, pages)
    got = idx.score_matrix(qbf)
    assert_scores(dtype, got, want, f"special values {dtype}, BF16 queries")
    assert_scores(dtype, idx.score_matrix(q32), want, f"special values {dtype}, F32 queries")
