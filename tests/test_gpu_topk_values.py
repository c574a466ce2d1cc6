"""b200ms_topk and b200ms_merge_topk on every value class and at the kernel-switch boundaries (run with -m gpu on an H100).

Score matrices are built on the host and handed to the C-ABI directly.  The oracle (oracle/maxsim_oracle.rank_desc_np) is
the documented total order: score DESC then id ASC, -0 == +0, every NaN above every number and NaNs tied.  Sums are formed
as the header says (groups in order from +0.0f in float32; for I32 scores in int64, clamped to +-(2^31 - 1)), and a
reported score is float32(sum) * scale in fp32 -- compared bit for bit, a NaN as 0x7fffffff.  The I32 class "overflow"
has sums past +-2^31: every group at INT32_MAX or INT32_MIN, alternating signs, sums exactly at +-(2^31 - 1), one past
it and 2^31 - 2, so that a wrapped, truncated or misplaced bound changes the order.

Boundaries: n_pages 1024 / 1025 (counting kernel vs radix select), multiples of 8192 (slice count), k at and around the
slice cap 8192 / k, k above the number of allowed pages; columns past n_pages (ld > n_pages) hold sentinels that would
rank first if they were read; allow-mask bits past n_pages are set and must be ignored.
"""
import ctypes
import functools

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

torch = pytest.importorskip("torch")
if not torch.cuda.is_available():  # pragma: no cover - the gpu marker normally deselects these on CPU boxes
    pytest.skip("CUDA device required", allow_module_level=True)

from morphik_core_b200 import _native as nat  # noqa: E402
from oracle import maxsim_oracle as orc  # noqa: E402
from oracle.scoring import i32_sum  # noqa: E402

F32 = np.float32
INT_MAX = (1 << 31) - 1
ID_BASE = 1 << 40
N_PAGES = [1, 1023, 1024, 1025, 8191, 8192, 16383, 16384, 16385, 64 * 8192 + 5]
KS = [1, 7, 1024, 1025, 2048, 2049, 2731, 4096]
CANON_NAN = np.uint32(0x7FFFFFFF)


@pytest.fixture(scope="module")
def h():
    return nat.Handle(0)


def vp(t):
    return ctypes.c_void_p(t.data_ptr()) if t is not None else None


def stream():
    return ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)


def bits_of(x):
    """float32 bit patterns with every NaN as the canonical 0x7fffffff."""
    x = np.asarray(x, F32)
    b = x.view(np.uint32).copy()
    b[np.isnan(x)] = CANON_NAN
    return b


# ------------------------------------------------------------------------------------------------ value classes
def nan_patterns(rng, n):
    """NaNs of both signs with random payloads."""
    payload = rng.integers(1, 1 << 23, size=n, dtype=np.uint64).astype(np.uint32)
    sign = rng.integers(0, 2, size=n, dtype=np.uint64).astype(np.uint32) << np.uint32(31)
    return (np.uint32(0x7F800000) | payload | sign).view(F32)


def f32_class(name, rng, shape):
    n = int(np.prod(shape))
    if name == "equal":
        v = np.full(n, 0.375, F32)
    elif name == "two":
        v = rng.choice(np.asarray([1.0, 2.0], F32), size=n)
    elif name == "zeros":
        v = rng.choice(np.asarray([0.0, -0.0, 1.0, -1.0], F32), size=n, p=[0.4, 0.4, 0.1, 0.1])
    elif name == "inf":  # inf + -inf across groups makes NaN sums too
        v = rng.choice(np.asarray([np.inf, -np.inf, 3.0, -3.0], F32), size=n)
    elif name == "subnormal":
        mag = rng.integers(0, 1 << 23, size=n, dtype=np.uint64).astype(np.uint32) % np.uint32(64)  # few values: ties
        v = (mag | (rng.integers(0, 2, size=n, dtype=np.uint64).astype(np.uint32) << np.uint32(31))).view(F32)
    elif name == "nan":
        v = rng.standard_normal(n).astype(F32)
        m = rng.random(n) < 0.3
        v[m] = nan_patterns(rng, int(m.sum()))
        v[rng.random(n) < 0.05] = np.inf
    elif name == "gauss":
        v = rng.standard_normal(n).astype(F32)
    else:
        raise ValueError(name)
    return v.reshape(shape)


F32_CLASSES = ["equal", "two", "zeros", "inf", "subnormal", "nan", "gauss"]
I32_CLASSES = ["equal", "two", "extremes", "large", "overflow"]
GROUPS = {"overflow": 4}  # groups of a class's query (default (i % 4) + 1)
INT_MIN = -(1 << 31)
# group scores of the "overflow" class (4 groups): sums beyond +-(2^31 - 1), at it, one past it and next to it
OVERFLOW_ROWS = np.asarray([
    [INT_MAX, INT_MAX, INT_MAX, INT_MAX], [INT_MIN, INT_MIN, INT_MIN, INT_MIN], [INT_MAX, 0, 0, 0], [INT_MAX - 1, 0, 0, 0],
    [INT_MAX - 3, 1, 1, 1], [INT_MAX - 3, 1, 1, 2], [INT_MAX, 1, 0, 0], [1 << 30, 1 << 30, 0, 0], [1 << 30, 1 << 30, -1, 0],
    [INT_MIN, 0, 0, 0], [-INT_MAX, 0, 0, 0], [-INT_MAX + 1, 0, 0, 0], [INT_MIN, 1, 0, 0], [INT_MIN, -1, 0, 0],
    [INT_MAX, -INT_MAX, INT_MAX, -INT_MAX], [INT_MAX, INT_MAX, INT_MIN, INT_MIN], [INT_MAX, INT_MAX, INT_MAX, INT_MIN],
    [INT_MIN, INT_MIN, INT_MAX, 5], [(1 << 24) + 1, 0, 0, 0], [1 << 24, 0, 0, 0], [12345, 0, 0, 0]], np.int64)


def split_sum(rng, total, parts):
    """int64 [n] totals -> [parts, n] int32 summands whose prefix sums stay between 0 and the total (no int32 overflow)."""
    total = np.asarray(total, np.int64)
    cuts = np.sort(rng.random((parts - 1, total.size)), axis=0)
    bounds = np.concatenate([np.zeros((1, total.size)), cuts, np.ones((1, total.size))])
    prefix = np.floor(bounds * total).astype(np.int64)
    prefix[-1] = total
    return np.diff(prefix, axis=0).astype(np.int32)


def i32_class(name, rng, groups, n):
    if name == "overflow":  # summands that pass int32 on their own
        parts = OVERFLOW_ROWS[rng.integers(0, len(OVERFLOW_ROWS), size=n)].T
        assert parts.shape[0] == groups
        return parts.astype(np.int32), parts.sum(axis=0)
    if name == "equal":
        tot = np.full(n, 12345, np.int64)
    elif name == "two":
        tot = rng.choice(np.asarray([-5, 7], np.int64), size=n)
    elif name == "extremes":  # sums of exactly INT_MAX and INT_MIN + 1, and neighbours
        tot = rng.choice(np.asarray([INT_MAX, INT_MAX - 1, -INT_MAX, -INT_MAX + 1, 0], np.int64), size=n)
    elif name == "large":  # above 2^24: float32 merges neighbours, the key must not
        tot = (1 << 24) + rng.integers(0, 64, size=n) * rng.choice(np.asarray([1, -1], np.int64), size=n) + \
            rng.choice(np.asarray([0, 1 << 28], np.int64), size=n)
    else:
        raise ValueError(name)
    return split_sum(rng, tot, groups), tot


# ------------------------------------------------------------------------------------------------ b200ms_topk
class Case:
    """One score matrix: a query per value class, query i summing (i % 4) + 1 groups; columns past n_pages hold sentinels."""

    def __init__(self, dtype, n_pages, seed):
        rng = np.random.default_rng(seed)
        self.dtype, self.n_pages = dtype, n_pages
        self.ld = n_pages + 37
        classes = F32_CLASSES if dtype == "f32" else I32_CLASSES
        self.ngroups = [GROUPS.get(name, (i % 4) + 1) for i, name in enumerate(classes)]
        self.goff = np.concatenate([[0], np.cumsum(self.ngroups)]).astype(np.int32)
        G = int(self.goff[-1])
        if dtype == "f32":
            gs = np.empty((G, self.ld), F32)
            gs[:, n_pages:] = nan_patterns(rng, G * 37).reshape(G, 37)  # would rank above everything if read
        else:
            gs = np.full((G, self.ld), INT_MAX, np.int32)
        self.sums = []
        for q, name in enumerate(classes):
            g0, g1 = self.goff[q], self.goff[q + 1]
            if dtype == "f32":
                gs[g0:g1, :n_pages] = f32_class(name, rng, (g1 - g0, n_pages))
                acc = np.zeros(n_pages, F32)  # +0.0f, groups in order, float32
                with np.errstate(invalid="ignore", over="ignore"):
                    for g in range(g0, g1):
                        acc = acc + gs[g, :n_pages]
                self.sums.append(acc)
            else:
                parts, tot = i32_class(name, rng, g1 - g0, n_pages)
                gs[g0:g1, :n_pages] = parts
                assert np.array_equal(parts.astype(np.int64).sum(axis=0), tot)
                self.sums.append(i32_sum(tot))  # the I32 sum rule: int64, clamped to +-(2^31 - 1)
        self.scale = F32(1.0) if dtype == "f32" else F32(1.0 / (127.0 * 127.0))
        self.gs = torch.from_numpy(gs).cuda()
        self.classes = classes
        self._order = {}

    def order(self, q, mask_name, allow):
        """Oracle order of query q's allowed pages (full length; a top-k is its prefix)."""
        key = (q, mask_name)
        if key not in self._order:
            ids = np.arange(self.n_pages, dtype=np.int64) if allow is None else np.flatnonzero(allow)
            self._order[key] = ids[orc.rank_desc_np(self.sums[q][ids], ids)]
        return self._order[key]

    def reported(self, q, ids):
        s = self.sums[q][ids]
        return bits_of(s.astype(F32) * self.scale)  # float32(sum) * scale in fp32


def masks(n_pages, rng):
    """name -> (bool allow per page or None, device uint32 words); the words carry set bits past n_pages."""
    words = (n_pages + 31) // 32 + 2
    out = {"none": (None, None)}
    out["zero"] = (np.zeros(n_pages, bool), np.zeros(words, np.uint32))
    every = np.arange(n_pages) % 32 == 5
    out["every32"] = (every, None)
    half = rng.random(n_pages) < 0.5
    out["half"] = (half, None)
    res = {}
    for name, (allow, w) in out.items():
        if allow is not None and w is None:
            bits = np.ones(words * 32, bool)  # everything past n_pages allowed: must be ignored
            bits[:n_pages] = allow
            w = (bits.reshape(-1, 32).astype(np.uint64) << np.arange(32, dtype=np.uint64)).sum(axis=1).astype(np.uint32)
        res[name] = (allow, None if w is None else torch.from_numpy(w.view(np.int32)).cuda())
    return res


@functools.lru_cache(maxsize=None)
def case(dtype, n_pages):
    return Case(dtype, n_pages, seed=n_pages * 2 + (dtype == "i32"))


@pytest.mark.parametrize("n_pages", N_PAGES)
@pytest.mark.parametrize("dtype", ["f32", "i32"])
def test_topk_every_value_class_and_boundary(h, dtype, n_pages):
    c = case(dtype, n_pages)
    n_q = len(c.classes)
    goff = nat.i32_array(c.goff.tolist())
    sdt = nat.F32 if dtype == "f32" else nat.I32
    mk = masks(n_pages, np.random.default_rng(n_pages))
    for mask_name, (allow, words) in mk.items():
        for k in KS:
            if mask_name != "none" and k not in (1, 1025, 2731, 4096):
                continue  # masks on a subset of k: the selection paths are the same
            ts = torch.full((n_q, k), 123.0, dtype=torch.float32, device="cuda")  # outputs are [n_q, k]
            ti = torch.full((n_q, k), -7, dtype=torch.int64, device="cuda")
            tc = torch.full((n_q,), -7, dtype=torch.int32, device="cuda")
            h.check(nat.lib.b200ms_topk(h.ptr, vp(c.gs), sdt, n_pages, c.ld, goff, n_q, vp(words), k, ctypes.c_float(c.scale),
                                        ID_BASE, vp(ts), vp(ti), vp(tc), stream()), "b200ms_topk")
            torch.cuda.synchronize()
            gs_, gi, gc = ts.cpu().numpy(), ti.cpu().numpy(), tc.cpu().numpy()
            for q in range(n_q):
                what = f"{dtype} n_pages={n_pages} k={k} mask={mask_name} class={c.classes[q]}"
                want = c.order(q, mask_name, allow)[:k]
                n = len(want)
                assert gc[q] == n, (what, gc[q], n)
                bad = np.flatnonzero(gi[q, :n] != want + ID_BASE)
                assert not len(bad), (what, bad[:5], gi[q, bad[:5]] - ID_BASE, want[bad[:5]])
                got_bits = bits_of(gs_[q, :n])
                want_bits = c.reported(q, want)
                bad = np.flatnonzero(got_bits != want_bits)
                assert not len(bad), (what, bad[:5], got_bits[bad[:5]], want_bits[bad[:5]])
                assert np.all(gi[q, n:] == -1) and np.all(np.isneginf(gs_[q, n:])), what


# ------------------------------------------------------------------------------------------------ b200ms_merge_topk
MS = [1, 2, 3, 1000, 4097, 8192]
MERGE_CLASSES = ["equal", "two", "zeros", "inf", "subnormal", "nan", "gauss", "all_invalid"]


def merge_ks(m):
    return sorted({k for k in (1, m - 1, m, m + 1, 4096) if 1 <= k <= nat.MAX_K})


@pytest.mark.parametrize("m", MS)
def test_merge_topk_every_value_class(h, m):
    rng = np.random.default_rng(m)
    n_q = len(MERGE_CLASSES)
    s = np.empty((n_q, m), F32)
    ids = np.empty((n_q, m), np.int64)
    for q, name in enumerate(MERGE_CLASSES):
        s[q] = f32_class("nan" if name == "all_invalid" else name, rng, (m,))
        ids[q] = rng.integers(0, 1 << 62, size=m, dtype=np.int64)  # ids up to 2^62 ...
        small = rng.random(m) < 0.3
        ids[q, small] = rng.integers(0, 4, size=int(small.sum()))  # ... and a few small ones, repeated: equal scores and ids
        ids[q, rng.random(m) < 0.1] = -1  # ignored
        if name == "all_invalid":
            ids[q] = -1
    sd, idd = torch.from_numpy(s).cuda(), torch.from_numpy(ids).cuda()
    for k in merge_ks(m):
        ts = torch.full((n_q, k), 123.0, dtype=torch.float32, device="cuda")
        ti = torch.full((n_q, k), -7, dtype=torch.int64, device="cuda")
        tc = torch.full((n_q,), -7, dtype=torch.int32, device="cuda")
        h.check(nat.lib.b200ms_merge_topk(h.ptr, vp(sd), vp(idd), n_q, m, k, vp(ts), vp(ti), vp(tc), stream()),
                "b200ms_merge_topk")
        torch.cuda.synchronize()
        gs_, gi, gc = ts.cpu().numpy(), ti.cpu().numpy(), tc.cpu().numpy()
        for q, name in enumerate(MERGE_CLASSES):
            what = f"merge m={m} k={k} class={name}"
            valid = np.flatnonzero(ids[q] >= 0)
            order = valid[orc.rank_desc_np(s[q, valid], ids[q, valid])][:k]
            n = len(order)
            assert gc[q] == n, (what, gc[q], n)
            # entries with equal (score, id) are interchangeable: compare ids and canonical scores position by position
            bad = np.flatnonzero(gi[q, :n] != ids[q, order])
            assert not len(bad), (what, bad[:5], gi[q, bad[:5]], ids[q, order][bad[:5]], s[q, order][bad[:5]])
            with np.errstate(invalid="ignore"):
                want_bits = bits_of(s[q, order] + F32(0.0))  # -0 reported as +0, NaN canonical
            got_bits = bits_of(gs_[q, :n])
            bad = np.flatnonzero(got_bits != want_bits)
            assert not len(bad), (what, bad[:5], got_bits[bad[:5]], want_bits[bad[:5]])
            assert np.all(gi[q, n:] == -1) and np.all(np.isneginf(gs_[q, n:])), what


# ------------------------------------------------------------------------------------------------ which kernels run
def kernels_launched(fn):
    from torch.profiler import ProfilerActivity, profile

    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    return [e.name for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA]


@pytest.mark.parametrize("n_pages,k,want", [(1024, 7, {"topk_small_kernel"}), (1025, 7, {"topk_kernel"}),
                                             (16383, 7, {"topk_kernel"}), (16384, 7, {"topk_kernel", "merge_topk_kernel"}),
                                             (16384, 4096, {"topk_kernel", "merge_topk_kernel"}),
                                             (64 * 8192 + 5, 2731, {"topk_kernel", "merge_topk_kernel"})])
def test_topk_dispatch_boundaries(h, n_pages, k, want):
    """The boundaries the value tests sit on are the real ones: up to 1024 pages the counting kernel, above it the radix
    select, and from 2 * 8192 pages on (while 8192 / k allows two slices) the sliced select plus the merge.  The results
    of the paths agree by design, so only the launched kernels show a moved boundary."""
    c = case("f32", n_pages) if n_pages in N_PAGES else Case("f32", n_pages, seed=5)
    n_q = len(c.classes)
    ts = torch.empty((n_q, k), dtype=torch.float32, device="cuda")
    ti = torch.empty((n_q, k), dtype=torch.int64, device="cuda")
    tc = torch.empty((n_q,), dtype=torch.int32, device="cuda")
    goff = nat.i32_array(c.goff.tolist())

    def run():
        h.check(nat.lib.b200ms_topk(h.ptr, vp(c.gs), nat.F32, n_pages, c.ld, goff, n_q, None, k, ctypes.c_float(1.0), 0,
                                    vp(ts), vp(ti), vp(tc), stream()), "b200ms_topk")

    run()  # warm (first-use attribute setting is not a launch we look at)
    names = kernels_launched(run)
    got = {next(n for n in ("merge_topk_kernel", "topk_small_kernel", "topk_kernel") if n in x) for x in names if "topk" in x}
    assert got == want, (n_pages, k, names)
