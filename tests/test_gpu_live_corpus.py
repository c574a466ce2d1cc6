"""A live HBM corpus: growable device blocks, compaction in place, and the indexes built on both (run with -m gpu on an H100).

  * b200ms_compact_rows against torch.cat of the runs, bit for bit: the run patterns of tests/test_compact_plan_cpu.py for
    every row size the product uses (16 / 128 / 256 bytes of patch rows, 20480 of an FDE row), and a buffer of 3 GiB whose
    walk is hundreds of grid waves deep, with bounce and direct windows.
  * b200ms_block_*: contents and address survive growing, a shrink hands the memory back to the driver, refusals, and out of
    memory without taking memory from anyone.
  * MaxSimIndex / TwoStageIndex: an index grown page by page equals one sized up front; a compacted index equals one built
    from the kept pages alone -- rows, scores, top-k.
  * Shard files on both tiers, fresh and appended to an index, empty ones too: read into the index's own block, equal to
    the index they were saved from.
  * Free device memory around growth and compaction, and around a store's open / load: the block lives outside torch's
    allocator, so the tests sample the device memory this process holds, through NVML's per-process accounting, which
    other jobs on the card do not move (torch.cuda.mem_get_info's free memory where NVML cannot tell this process apart).
    The bounds carry a tolerance of 256 MiB.
  * One stream-order case: a search in flight on one stream, a compaction, a search after it.
"""
import asyncio
import ctypes

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

torch = pytest.importorskip("torch")
if not torch.cuda.is_available():  # pragma: no cover - the gpu marker normally deselects these on CPU boxes
    pytest.skip("CUDA device required", allow_module_level=True)

import compact_model as cm  # noqa: E402
from morphik_core_b200 import _native as nat  # noqa: E402
from morphik_core_b200 import shardfile  # noqa: E402
from morphik_core_b200.fde import FixedDimensionalEncodingConfig, TwoStageIndex  # noqa: E402
from morphik_core_b200.index import DeviceBlock, MaxSimIndex, _aligned_bytes  # noqa: E402
from morphik_core_b200.models import DocumentChunk  # noqa: E402
from morphik_core_b200.store import B200MultiVectorStore  # noqa: E402
from test_compact_plan_cpu import page_runs, patterns  # noqa: E402

DEV = torch.device("cuda", 0)
CHUNK = 32 << 20
TOL = 256 << 20  # scratch the handle keeps, and other jobs on the card where free_bytes cannot exclude them
DTYPES = ("bf16", "int8", "fp8", "binary")


def i64p(a):
    return a.ctypes.data_as(nat.i64p)


def cstream():
    return ctypes.c_void_p(torch.cuda.current_stream(DEV).cuda_stream)


def _nvml_own_pid():
    """This process's pid as NVML reports it (it may differ from os.getpid() inside a container): the one process whose
    device memory grows by a 256 MiB block backed for the purpose.  None when NVML cannot say (no NVML, no per-process
    accounting, or another process grew as much at the same time)."""
    try:
        import pynvml

        pynvml.nvmlInit()
        dev = pynvml.nvmlDeviceGetHandleByIndex(DEV.index or 0)

        def used():
            torch.cuda.synchronize(DEV)
            return {p.pid: p.usedGpuMemory for p in pynvml.nvmlDeviceGetComputeRunningProcesses(dev)}

        h = nat.Handle(DEV.index or 0)
        try:
            before = used()
            probe = DeviceBlock.resized(None, h, DEV, 256 << 20)
            after = used()
            probe.free()
        finally:
            torch.cuda.synchronize(DEV)
            h.close()
        grown = [pid for pid, u in after.items() if u is not None and u - (before.get(pid) or 0) >= (192 << 20)]
        return (dev, grown[0]) if len(grown) == 1 else None
    except Exception:  # pragma: no cover - NVML missing or refused: fall back to the card's free memory
        return None


_OWN = []


def free_bytes():
    """Device memory free to this process: the card's total less what this process holds (NVML's per-process use), so
    that other jobs on the card move none of the bounds below; torch.cuda.mem_get_info's free memory, and the bounds'
    tolerance, where NVML cannot tell this process apart."""
    if not _OWN:
        _OWN.append(_nvml_own_pid())
    torch.cuda.synchronize(DEV)
    free, total = torch.cuda.mem_get_info(DEV)
    if _OWN[0] is None:
        return free
    import pynvml

    dev, pid = _OWN[0]
    mine = [p.usedGpuMemory for p in pynvml.nvmlDeviceGetComputeRunningProcesses(dev) if p.pid == pid]
    assert len(mine) == 1 and mine[0] is not None, "NVML lost track of this process"
    return total - mine[0]


@pytest.fixture(scope="module")
def handle():
    h = nat.Handle(0)
    yield h
    torch.cuda.synchronize(DEV)
    h.close()


def compact_rows(h, buf, row_bytes, run_start, run_rows):
    rs, rr = np.asarray(run_start, dtype=np.int64), np.asarray(run_rows, dtype=np.int64)
    return nat.lib.b200ms_compact_rows(h.ptr, ctypes.c_void_p(buf.data_ptr()), row_bytes, i64p(rs), i64p(rr), len(rs), cstream())


def check_compaction(h, n_rows, row_bytes, run_start, run_rows, seed=0):
    g = torch.Generator(device=DEV)
    g.manual_seed(seed)
    buf = torch.randint(0, 256, (n_rows, row_bytes), dtype=torch.uint8, device=DEV, generator=g)
    parts = [buf[s:s + n] for s, n in zip(run_start, run_rows)]
    want = torch.cat(parts).clone() if parts else buf[:0].clone()
    h.check(compact_rows(h, buf, row_bytes, run_start, run_rows), "b200ms_compact_rows")
    torch.cuda.synchronize(DEV)
    assert torch.equal(buf[: want.shape[0]], want)


# ------------------------------------------------------------------------------------------------ compaction kernel
@pytest.mark.parametrize("row_bytes", [16, 128, 256, 20480])
@pytest.mark.parametrize("name", sorted(patterns(8)))
def test_compact_rows_equals_cat_of_the_runs(handle, name, row_bytes):
    """160 MiB in 1280 pages of 128 KiB (200 MiB in 160 pages of 64 FDE-sized rows), so the walk crosses several 64 MiB
    windows whatever the row size; the model says which kinds of window the pattern takes."""
    page_rows, n_pages = (64, 160) if row_bytes == 20480 else ((128 << 10) // row_bytes, 1280)
    rs, rr = page_runs(patterns(n_pages)[name], page_rows)
    windows = cm.compact_in_place(np.zeros(n_pages * page_rows, dtype=np.uint8), 1, rs, rr, *cm.library_windows(row_bytes))
    if name in ("first_page_deleted", "one_hole", "alternating"):
        assert len(windows) >= 2 and "bounce" in {k for _, _, k in windows}, windows
    if name in ("alternating", "first_half_deleted"):
        assert "direct" in {k for _, _, k in windows}, windows
    check_compaction(handle, n_pages * page_rows, row_bytes, rs, rr)


def test_compact_rows_ragged_runs_and_empty_runs(handle):
    rng = np.random.default_rng(3)
    n_rows = 1 << 20
    cuts = np.sort(rng.choice(n_rows + 1, size=20000, replace=False))
    rs, rr = [int(a) for a in cuts[0::2]], [int(b - a) for a, b in zip(cuts[0::2], cuts[1::2])]
    rs.insert(1, rs[0] + rr[0]); rr.insert(1, 0)
    check_compaction(handle, n_rows, 128, rs, rr)


def test_compact_rows_three_gib(handle):
    """3 GiB of 256-byte rows in pages of 1024 rows: (a) only the first page deleted -- every row moves by one page, 48
    bounce windows; (b) 30 % of the pages deleted singly -- thousands of short runs, bounce windows first, then direct ones
    of growing size.  Checked without a second 3 GiB copy: row r of the buffer holds r in its first 8 bytes, a multiple
    of r in the next 8 and ~r in its last 8, and the rest is zero."""
    page_rows, n_pages, row_bytes = 1024, 12288, 256
    n_rows = page_rows * n_pages
    rng = np.random.default_rng(11)
    for keep in (list(range(1, n_pages)), [p for p in range(n_pages) if rng.random() >= 0.3]):
        buf = torch.zeros((n_rows, row_bytes // 8), dtype=torch.int64, device=DEV)
        buf[:, 0] = torch.arange(n_rows, device=DEV)
        buf[:, 1] = buf[:, 0] * 2654435761
        buf[:, 31] = ~buf[:, 0]
        rs, rr = page_runs(keep, page_rows)
        kinds = [k for _, _, k in cm.compact_in_place(np.zeros(n_rows, dtype=np.uint8), 1, rs, rr, *cm.library_windows(row_bytes))]
        assert kinds.count("bounce") >= (48 if len(rs) == 1 else 1) and ("direct" in kinds) == (len(rs) > 1)
        handle.check(compact_rows(handle, buf.view(torch.uint8), row_bytes, rs, rr), "b200ms_compact_rows")
        src = torch.from_numpy(np.concatenate([np.arange(s, s + n, dtype=np.int64) for s, n in zip(rs, rr)])).to(DEV)
        got = buf[: src.shape[0]]
        assert torch.equal(got[:, 0], src) and torch.equal(got[:, 1], src * 2654435761) and torch.equal(got[:, 31], ~src)
        assert not got[:, 2:31].any()
        del buf, got, src


def test_compact_rows_refusals(handle):
    buf = torch.zeros((64, 256), dtype=torch.uint8, device=DEV)
    before = nat.lib.b200ms_launch_count(handle.ptr)
    assert compact_rows(handle, buf, 24, [0], [1]) == -1  # row_bytes not a multiple of 16
    assert compact_rows(handle, buf, 0, [0], [1]) == -1
    assert compact_rows(handle, buf, 256, [4, 0], [2, 2]) == -1  # out of order
    assert compact_rows(handle, buf, 256, [0, 3], [4, 2]) == -1  # overlapping
    assert compact_rows(handle, buf, 256, [0], [-1]) == -1
    assert compact_rows(handle, buf[0, 8:], 16, [1], [1]) == -1  # not 16-byte aligned
    assert nat.lib.b200ms_compact_rows(handle.ptr, None, 256, None, None, 1, cstream()) == -1
    assert compact_rows(handle, buf, 256, [], []) == 0
    assert nat.lib.b200ms_launch_count(handle.ptr) == before  # nothing was launched


# ------------------------------------------------------------------------------------------------ blocks
def new_block(h, max_bytes):
    p = ctypes.c_void_p()
    h.check(nat.lib.b200ms_block_create(h.ptr, max_bytes, ctypes.byref(p)), "b200ms_block_create")
    return p


def block_tensor(p):
    from morphik_core_b200.index import _CudaBytes

    return torch.as_tensor(_CudaBytes(nat.lib.b200ms_block_ptr(p), nat.lib.b200ms_block_mapped_bytes(p)), device=DEV)


def test_block_grows_in_place_and_returns_memory(handle):
    g = torch.Generator(device=DEV)
    g.manual_seed(1)
    data = torch.randint(0, 256, (1 << 30,), dtype=torch.uint8, device=DEV, generator=g)
    torch.cuda.empty_cache()  # what torch caches is not free to the driver
    start = free_bytes()
    p = new_block(handle, 8 << 30)
    base = nat.lib.b200ms_block_ptr(p)
    assert base and base % 1024 == 0 and nat.lib.b200ms_block_mapped_bytes(p) == 0
    assert abs(free_bytes() - start) <= TOL  # address space only
    filled = 0
    for size in (1, CHUNK, CHUNK + 1, 200 << 20, 1 << 30):  # bytes asked for; whole chunks are backed
        handle.check(nat.lib.b200ms_block_resize(handle.ptr, p, size), "b200ms_block_resize")
        assert nat.lib.b200ms_block_mapped_bytes(p) == -(-size // CHUNK) * CHUNK and nat.lib.b200ms_block_ptr(p) == base
        t = block_tensor(p)
        assert t.data_ptr() == base and t.device == DEV
        assert torch.equal(t[:filled], data[:filled])  # what was there stays
        t[filled:size].copy_(data[filled:size])
        filled = size
    mapped = free_bytes()
    assert abs((start - mapped) - (1 << 30)) <= TOL
    handle.check(nat.lib.b200ms_block_resize(handle.ptr, p, 100 << 20), "b200ms_block_resize")
    assert nat.lib.b200ms_block_mapped_bytes(p) == 128 << 20
    assert abs((free_bytes() - mapped) - ((1 << 30) - (128 << 20))) <= TOL  # the tail is back with the driver, not cached
    assert torch.equal(block_tensor(p)[: 100 << 20], data[: 100 << 20])
    handle.check(nat.lib.b200ms_block_resize(handle.ptr, p, 0), "b200ms_block_resize")
    assert nat.lib.b200ms_block_mapped_bytes(p) == 0
    handle.check(nat.lib.b200ms_block_resize(handle.ptr, p, 3 * CHUNK), "b200ms_block_resize")
    t = block_tensor(p)
    t.copy_(data[: 3 * CHUNK])
    assert torch.equal(t, data[: 3 * CHUNK])
    del t
    handle.check(nat.lib.b200ms_block_destroy(handle.ptr, p), "b200ms_block_destroy")
    assert abs(free_bytes() - start) <= TOL


def test_block_out_of_memory_takes_nothing(handle):
    """A request that cannot fit is refused from cudaMemGetInfo's answer, before any physical memory is created."""
    total = torch.cuda.get_device_properties(DEV).total_memory
    p = new_block(handle, total + (1 << 30))
    handle.check(nat.lib.b200ms_block_resize(handle.ptr, p, 2 * CHUNK), "b200ms_block_resize")
    t = block_tensor(p)
    data = torch.arange(2 * CHUNK, device=DEV, dtype=torch.int32).to(torch.uint8)
    t.copy_(data)
    before = free_bytes()
    assert nat.lib.b200ms_block_resize(handle.ptr, p, total + (1 << 30)) == -4  # B200MS_ENOMEM
    assert b"do not fit" in nat.lib.b200ms_last_error(handle.ptr)
    assert nat.lib.b200ms_block_mapped_bytes(p) == 2 * CHUNK
    assert abs(free_bytes() - before) <= TOL
    assert torch.equal(t, data)
    handle.check(nat.lib.b200ms_block_resize(handle.ptr, p, 3 * CHUNK), "b200ms_block_resize")  # and it still grows
    del t
    handle.check(nat.lib.b200ms_block_destroy(handle.ptr, p), "b200ms_block_destroy")


def test_block_refusals(handle):
    other = nat.Handle(0)
    p = new_block(handle, 4 * CHUNK)
    out = ctypes.c_void_p()
    assert nat.lib.b200ms_block_create(handle.ptr, -1, ctypes.byref(out)) == -1
    assert nat.lib.b200ms_block_create(handle.ptr, CHUNK, None) == -1
    assert nat.lib.b200ms_block_resize(handle.ptr, p, -1) == -1
    assert nat.lib.b200ms_block_resize(handle.ptr, p, 4 * CHUNK + 1) == -1
    assert nat.lib.b200ms_block_resize(handle.ptr, None, 0) == -1
    assert nat.lib.b200ms_block_resize(other.ptr, p, CHUNK) == -1  # a block of another handle
    assert nat.lib.b200ms_block_destroy(other.ptr, p) == -1
    assert nat.lib.b200ms_block_mapped_bytes(p) == 0
    handle.check(nat.lib.b200ms_block_resize(handle.ptr, p, 4 * CHUNK), "b200ms_block_resize")
    handle.check(nat.lib.b200ms_block_destroy(handle.ptr, p), "b200ms_block_destroy")
    # a forgotten block goes with its handle
    start = free_bytes()
    q = new_block(other, 8 * CHUNK)
    other.check(nat.lib.b200ms_block_resize(other.ptr, q, 8 * CHUNK), "b200ms_block_resize")
    other.close()
    assert abs(free_bytes() - start) <= TOL


# ------------------------------------------------------------------------------------------------ indexes
def make_pages(n_pages, seed, lo=1, hi=300):
    g = torch.Generator(device=DEV)
    g.manual_seed(seed)
    rng = np.random.default_rng(seed)
    lens = [int(x) for x in rng.integers(lo, hi, size=n_pages)]
    lens[3] = 0
    rows = torch.randn((sum(lens), nat.DIM), generator=g, device=DEV)
    rows = rows / rows.norm(dim=1, keepdim=True)
    return list(rows.split(lens))


def make_queries(seed, lens=(32, 20, 40, 7)):
    g = torch.Generator(device=DEV)
    g.manual_seed(seed)
    return [torch.randn((t, nat.DIM), generator=g, device=DEV) for t in lens]


def search(idx, queries, k=10):
    q = torch.cat(queries).contiguous()
    ts, ti, tc = idx.search_device(q, [int(x.shape[0]) for x in queries], k)
    torch.cuda.synchronize(DEV)
    return ts.cpu(), ti.cpu(), tc.cpu()


def assert_same_index(a, b, queries):
    assert a.n_pages == b.n_pages and a.n_rows_padded == b.n_rows_padded
    assert torch.equal(a.packed_rows(), b.packed_rows())
    assert np.array_equal(a.score_matrix(queries), b.score_matrix(queries))
    for x, y in zip(search(a, queries), search(b, queries)):
        assert torch.equal(x, y)


@pytest.mark.parametrize("dtype", DTYPES)
def test_index_grown_in_small_steps_equals_index_reserved_once(dtype):
    """Pages of 2048..4096 rows, eight per call: the bf16 corpus (~800 MiB) grows by a chunk in every fifth call or so."""
    pages = make_pages(1024, seed=21, lo=2048, hi=4096)
    queries = make_queries(22)
    grown = MaxSimIndex(dtype=dtype)
    grows = 0
    for i in range(0, len(pages), 8):
        cap = grown._cap_rows
        grown.add_pages(pages[i:i + 8])
        grows += grown._cap_rows != cap
    assert grows >= (24 if dtype == "bf16" else 12 if dtype in ("int8", "fp8") else 2)
    once = MaxSimIndex(dtype=dtype)
    once.reserve_rows(grown.n_rows_padded)
    base = once._buf.data_ptr()
    once.add_pages(pages)
    assert once._buf.data_ptr() == base and base % 1024 == 0
    assert_same_index(grown, once, queries)
    grown.close()
    once.close()


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("pattern", ["first_page_deleted", "alternating", "random_30", "documents_30", "everything_deleted",
                                     "nothing_deleted"])
def test_compacted_index_equals_index_of_the_kept_pages(dtype, pattern):
    pages = make_pages(400, seed=31)
    queries = make_queries(32)
    keep = patterns(len(pages))[pattern]
    idx = MaxSimIndex(dtype=dtype)
    for i in range(0, len(pages), 50):
        idx.add_pages(pages[i:i + 50])
    search(idx, queries)  # attached and searched before the compaction
    base = idx._buf.data_ptr()
    idx.compact(keep)
    want = MaxSimIndex(dtype=dtype)
    want.add_pages([pages[p] for p in keep])
    if keep:
        assert idx._buf.data_ptr() == base
        assert_same_index(idx, want, queries)
    else:
        assert idx.n_pages == 0 and idx.packed_rows().shape == (0, idx.row_bytes)
    idx.add_pages(pages[:7])  # and it keeps growing afterwards
    want.add_pages(pages[:7])
    assert_same_index(idx, want, queries)
    idx.close()
    want.close()


def test_adopted_tensor_is_left_alone_by_growth_and_compaction():
    """adopt_packed stays zero-copy; the rows move into the index's own block when the index first grows or compacts."""
    src = MaxSimIndex(dtype="bf16")
    pages = make_pages(64, seed=41, lo=32, hi=33)
    pages[3] = pages[4]
    src.add_pages(pages)
    rows = _aligned_bytes(src.packed_rows().numel(), DEV).view(-1, 256)  # a caller's own 1024-byte aligned tensor
    rows.copy_(src.packed_rows())
    lens = [int(p.shape[0]) for p in pages]
    snapshot = rows.clone()
    for action in ("grow", "compact"):
        idx = MaxSimIndex(dtype="bf16")
        idx.adopt_packed(rows, lens)
        assert idx._buf.data_ptr() == rows.data_ptr() and idx._block is None
        if action == "grow":
            idx.add_pages(pages[:2])
            assert torch.equal(idx.packed_rows()[: rows.shape[0]], rows) and idx.n_pages == 66
        else:
            idx.compact(list(range(1, 64, 2)))
            assert torch.equal(idx.packed_rows(), rows.view(64, 32, 256)[1::2].reshape(-1, 256))
        assert isinstance(idx._block, DeviceBlock) and idx._buf.data_ptr() != rows.data_ptr()
        assert torch.equal(rows, snapshot)
        idx.close()
    src.close()


@pytest.mark.parametrize("pattern", ["alternating", "random_30", "first_page_deleted"])
def test_two_stage_index_grows_and_compacts_in_place(pattern):
    cfg = FixedDimensionalEncodingConfig(num_repetitions=8, num_simhash_projections=3, projection_dimension=8)
    pages = make_pages(300, seed=51)
    queries = make_queries(52)
    keep = patterns(len(pages))[pattern]
    two = TwoStageIndex(dtype="bf16", config=cfg)
    for i in range(0, len(pages), 20):
        two.add_pages(pages[i:i + 20])
    once = TwoStageIndex(dtype="bf16", config=cfg)
    once.add_pages(pages)
    for a, b in zip(two.fde_rows(), once.fde_rows()):
        assert torch.equal(a, b)
    base = two._F.data_ptr()
    two.compact(keep)
    want = TwoStageIndex(dtype="bf16", config=cfg)
    want.add_pages([pages[p] for p in keep])
    assert two.n_pages == want.n_pages == len(keep) and two._F.data_ptr() == base
    for a, b in zip(two.fde_rows(), want.fde_rows()):
        assert torch.equal(a, b)
    assert torch.equal(two.index.packed_rows(), want.index.packed_rows())
    for a, b in zip(two.search(queries, k=10, n_candidates=50), want.search(queries, k=10, n_candidates=50)):
        assert np.array_equal(a, b)
    two.add_pages(pages[:5])
    want.add_pages(pages[:5])
    for a, b in zip(two.search(queries, k=10, n_candidates=50), want.search(queries, k=10, n_candidates=50)):
        assert np.array_equal(a, b)
    for t in (two, once, want):
        t.index.close()


# ------------------------------------------------------------------------------------------------ shard files
def page_scores(idx, queries, tier):
    """What an index scores: score_matrix and search_device on the HBM tier, rerank_batch over every page on the host tier
    (the only search it has)."""
    if tier == "hbm":
        return [torch.from_numpy(idx.score_matrix(queries)), *search(idx, queries)]
    cand = torch.arange(idx.n_pages, device=DEV).repeat(len(queries), 1)
    out = idx.rerank_batch(torch.cat(queries).contiguous(), [int(x.shape[0]) for x in queries], cand, idx.n_pages)
    torch.cuda.synchronize(DEV)
    return [t.cpu() for t in out]


def assert_loaded(got, want, queries, tier):
    assert got.tier == tier
    assert torch.equal(got.packed_rows().cpu(), want.packed_rows().cpu())
    assert np.array_equal(got.page_lens, want.page_lens)
    for x, y in zip(page_scores(got, queries, tier), page_scores(want, queries, tier)):
        assert torch.equal(x, y)


@pytest.mark.parametrize("tier", ["hbm", "host"])
@pytest.mark.parametrize("dtype", DTYPES)
def test_shard_file_is_read_into_the_index_block(tmp_path, dtype, tier):
    """Loaded fresh and appended (into=) to an index that holds pages: the same rows, page lengths and scores as the
    index it was saved from; on HBM the rows sit in the index's DeviceBlock, which keeps its address as the index grows
    and compacts."""
    pages = make_pages(40, seed=81)  # one page of 0 rows, lengths that are not multiples of 32
    head = make_pages(9, seed=82)
    queries = make_queries(83)
    saved = MaxSimIndex(dtype=dtype)
    saved.add_pages(pages)
    path = str(tmp_path / "pages.b2ms")
    shardfile.save_index(saved, path)
    both = MaxSimIndex(dtype=dtype)
    both.add_pages(head + pages)
    fresh = shardfile.load_index(path, tier=tier)
    appended = MaxSimIndex(dtype=dtype, tier=tier)
    appended.add_pages(head)
    assert shardfile.load_index(path, into=appended) is appended
    assert_loaded(fresh, saved, queries, tier)
    assert_loaded(appended, both, queries, tier)
    if tier == "hbm":
        for idx in (fresh, appended):
            assert isinstance(idx._block, DeviceBlock)
            base = idx._buf.data_ptr()
            idx.add_pages(pages[:5])
            idx.compact(list(range(1, idx.n_pages, 2)))
            assert idx._buf.data_ptr() == base
    for idx in (saved, both, fresh, appended):
        idx.close()


@pytest.mark.parametrize("tier", ["hbm", "host"])
def test_empty_shard_file_loads_and_the_index_takes_pages(tmp_path, tier):
    path = str(tmp_path / "empty.b2ms")
    empty = MaxSimIndex(dtype="bf16")
    shardfile.save_index(empty, path)
    pages = make_pages(12, seed=91)
    queries = make_queries(92)
    want = MaxSimIndex(dtype="bf16")
    want.add_pages(pages)
    idx = shardfile.load_index(path, tier=tier)
    assert idx.n_pages == 0
    idx.add_pages(pages)
    shardfile.load_index(path, into=idx)
    assert_loaded(idx, want, queries, tier)
    for i in (empty, want, idx):
        i.close()


# ------------------------------------------------------------------------------------------------ free device memory
def test_growth_and_compaction_never_hold_a_second_copy():
    """1.5 GiB of bf16 rows ingested 64 MiB at a time, 30 % of its pages deleted, compacted.  Free device memory (sampled
    after every call, synchronised) never drops below start - corpus - one chunk - the pack call's temporaries (the float32
    source of 64 MiB of bf16 rows: 128 MiB), the compaction costs at most its bounce buffer, and afterwards the dead rows'
    bytes are back.  All within the tolerance for a shared card."""
    page_rows, pages_per_call, calls = 1024, 256, 24
    g = torch.Generator(device=DEV)
    g.manual_seed(61)
    batch = torch.randn((pages_per_call * page_rows, nat.DIM), generator=g, device=DEV)
    batch = list((batch / batch.norm(dim=1, keepdim=True)).split(page_rows))
    idx = MaxSimIndex(dtype="bf16")
    idx.add_pages(batch[:1])  # handle scratch and the first chunk exist before the baseline
    idx.clear()
    torch.cuda.empty_cache()
    start, torch_start = free_bytes(), torch.cuda.memory_allocated(DEV)
    lowest = start
    call_bytes = pages_per_call * page_rows * 256
    for i in range(calls):
        idx.add_pages(batch)
        free = free_bytes()
        lowest = min(lowest, free)
        assert start - free <= (i + 1) * call_bytes + CHUNK + 2 * call_bytes + TOL, i
    corpus = calls * call_bytes
    assert idx.n_rows_padded * 256 == corpus
    assert start - lowest <= corpus + CHUNK + 2 * call_bytes + TOL
    torch.cuda.empty_cache()
    full = free_bytes()
    rng = np.random.default_rng(62)
    keep = [p for p in range(idx.n_pages) if rng.random() >= 0.3]
    idx.compact(keep)
    after = free_bytes()
    dead = corpus - len(keep) * page_rows * 256
    bounce = 80 << 20  # the 64 MiB bounce buffer as the handle's scratch allocator rounds it; the handle keeps it
    assert dead - bounce - CHUNK - TOL <= after - full <= dead + TOL  # the dead rows are back with the driver
    assert torch.cuda.memory_allocated(DEV) - torch_start < corpus // 2  # and none of the corpus sits in torch's allocator
    idx.close()


def test_reopened_and_loaded_stores_never_hold_a_second_copy(tmp_path):
    """A durable bf16 store of 1.5 GiB, checkpointed as one base segment, then opened (journal replay), ingested into and
    compacted; and the same checkpoint loaded and ingested into.  The rows are read into the index's block: torch's
    allocator never holds more than an ingest call's temporaries, and free device memory (sampled after every call,
    synchronised) drops by at most the corpus, one chunk, the pack temporaries and the compaction's bounce buffer."""
    page_rows, pages_per_call, calls, per_doc = 1024, 1024, 6, 64
    g = torch.Generator(device=DEV)
    g.manual_seed(101)

    def chunks(first, n):
        rows = torch.randn((n * page_rows, nat.DIM), generator=g, device=DEV)
        rows = (rows / rows.norm(dim=1, keepdim=True)).bfloat16()
        return [DocumentChunk(document_id=f"d{(first + i) // per_doc}", content="", chunk_number=(first + i) % per_doc,
                              metadata={}, embedding=e) for i, e in enumerate(rows.split(page_rows))]

    d = str(tmp_path / "store")
    store = B200MultiVectorStore.open(d, mode="bf16")
    for c in range(calls):
        asyncio.run(store.store_embeddings(chunks(c * pages_per_call, pages_per_call)))
    store.save(d)
    store.close()
    corpus = calls * pages_per_call * page_rows * 256
    extra = chunks(calls * pages_per_call, per_doc)
    extra_bytes = per_doc * page_rows * 256
    bounce = 80 << 20  # the compaction's 64 MiB bounce buffer as the handle's scratch allocator rounds it
    for reopen in ("open", "load"):
        torch.cuda.empty_cache()
        start = free_bytes()
        torch.cuda.reset_peak_memory_stats(DEV)
        torch_start = torch.cuda.memory_allocated(DEV)
        if reopen == "open":
            store = B200MultiVectorStore.open(d, mode="bf16", compact_dead_fraction=0.0)
        else:
            store = B200MultiVectorStore.load(d)
        assert store._index.n_pages == calls * pages_per_call
        lowest = free_bytes()
        asyncio.run(store.store_embeddings(extra))
        lowest = min(lowest, free_bytes())
        if reopen == "open":
            assert asyncio.run(store.delete_chunks_by_document_id("d0"))  # any dead page compacts
            assert store._index.n_pages == calls * pages_per_call  # d0's pages are gone, the new document's are in
            lowest = min(lowest, free_bytes())
        assert torch.cuda.max_memory_allocated(DEV) - torch_start < corpus // 8, reopen
        assert start - lowest <= corpus + extra_bytes + CHUNK + 2 * extra_bytes + bounce + TOL, reopen
        store.close()


# ------------------------------------------------------------------------------------------------ stream order
def test_compaction_between_searches_on_different_streams():
    """A search enqueued on stream A, then compact on the current stream, then a search: both searches return what they return
    when run alone -- the compaction waits for the search that still reads the rows it is about to move and unmap."""
    pages = make_pages(6000, seed=71, lo=400, hi=620)  # ~780 MiB of bf16 rows: the first search is still running
    queries = make_queries(72, lens=[32] * 48)
    q = torch.cat(queries).contiguous()
    q_lens = [32] * 48
    rng = np.random.default_rng(73)
    keep = [p for p in range(len(pages)) if rng.random() >= 0.4]

    def build():
        idx = MaxSimIndex(dtype="bf16")
        idx.add_pages(pages)
        idx._attach()
        return idx

    alone = build()
    want_before = [t.clone() for t in alone.search_device(q, q_lens, 16)]
    torch.cuda.synchronize(DEV)
    alone.compact(keep)
    want_after = [t.clone() for t in alone.search_device(q, q_lens, 16)]
    torch.cuda.synchronize(DEV)
    alone.close()

    idx = build()
    torch.cuda.synchronize(DEV)
    side = torch.cuda.Stream(DEV)
    with torch.cuda.stream(side):
        got_before = idx.search_device(q, q_lens, 16)  # left in flight on the side stream
    idx.compact(keep)
    got_after = idx.search_device(q, q_lens, 16)
    torch.cuda.synchronize(DEV)
    for a, b in zip(got_before, want_before):
        assert torch.equal(a, b)
    for a, b in zip(got_after, want_after):
        assert torch.equal(a, b)
    idx.close()
