"""CPU checks of the in-place compaction (csrc/compact.cu) through its numpy restatement, tests/compact_model.py: the window
walk applied in place to a byte array must leave exactly what copying the surviving runs into a second buffer gives, and
must never read a row a launch has already overwritten.  Pages are 32 rows, as the smallest page of the packed layout, and
the windows are a few pages long so that every pattern crosses many of them; tests/test_gpu_live_corpus.py holds the kernel
to the same patterns.  Also here: the refusals of the new entry points that need no device."""
import ctypes

import numpy as np
import pytest

import compact_model as cm

PAGE = 32  # rows per page


def page_runs(keep, page_rows=PAGE):
    """Maximal runs of consecutive kept pages -> (run_start, run_rows) in rows."""
    starts, rows = [], []
    for p in keep:
        if starts and starts[-1] + rows[-1] == p * page_rows:
            rows[-1] += page_rows
        else:
            starts.append(p * page_rows)
            rows.append(page_rows)
    return starts, rows


def patterns(n_pages):
    rng = np.random.default_rng(n_pages)
    every = list(range(n_pages))
    return {
        "nothing_deleted": every,
        "everything_deleted": [],
        "first_page_deleted": every[1:],  # every row moves by one page: maximal overlap
        "last_page_deleted": every[:-1],
        "alternating": every[::2],
        "alternating_odd": every[1::2],
        "first_half_deleted": every[n_pages // 2:],  # one run larger than several windows, far from its destination
        "one_hole": every[:5] + every[6:],  # one run larger than several windows, one page from its destination
        "random_30": [p for p in every if rng.random() >= 0.3],
        "random_90": [p for p in every if rng.random() >= 0.9],
        "documents_30": [p for p in every if (p // 16) % 10 >= 3],
    }


def run_model(row_bytes, run_start, run_rows, n_rows, window_rows, min_direct_rows, max_direct_rows, seed=0):
    rng = np.random.default_rng(seed)
    buf = rng.integers(0, 256, size=n_rows * row_bytes, dtype=np.uint8)
    want = cm.out_of_place(buf.copy(), row_bytes, run_start, run_rows)
    before = buf.copy()
    windows = cm.compact_in_place(buf, row_bytes, run_start, run_rows, window_rows, min_direct_rows, max_direct_rows)
    got = buf.reshape(-1, row_bytes)
    assert np.array_equal(got[: len(want)], want)
    assert np.array_equal(got[len(want):], before.reshape(-1, row_bytes)[len(want):])  # nothing past the survivors is written
    return windows


@pytest.mark.parametrize("row_bytes", [16, 48])
@pytest.mark.parametrize("name", sorted(patterns(8)))
def test_window_walk_equals_out_of_place_copy(name, row_bytes):
    n_pages = 200
    keep = patterns(n_pages)[name]
    rs, rr = page_runs(keep)
    # windows of 3.5 pages straddle runs and pages; direct from 2 pages of displacement, at most 5 pages at a time
    windows = run_model(row_bytes, rs, rr, n_pages * PAGE, window_rows=112, min_direct_rows=64, max_direct_rows=160)
    kinds = {k for _, _, k in windows}
    if name in ("nothing_deleted", "everything_deleted", "last_page_deleted"):
        assert windows == []  # nothing moves
    if name in ("first_page_deleted", "one_hole"):
        assert kinds == {"bounce"} and len(windows) > 10  # one page of displacement never allows a direct window
    if name == "first_half_deleted":
        assert kinds == {"direct"} and len(windows) > 10
    if name == "alternating":
        assert kinds == {"bounce", "direct"}  # the displacement grows along the buffer
    if name in ("random_30", "documents_30"):
        assert "direct" in kinds
    assert all(a[0] + a[1] == b[0] for a, b in zip(windows, windows[1:]))  # ascending, no gap, no overlap


def test_random_run_sets_and_window_sizes():
    rng = np.random.default_rng(5)
    for trial in range(200):
        n_rows = int(rng.integers(1, 3000))
        cuts = np.sort(rng.choice(n_rows + 1, size=min(n_rows + 1, int(rng.integers(0, 40)) * 2), replace=False))
        rs, rr = [int(a) for a in cuts[0::2]], [int(b - a) for a, b in zip(cuts[0::2], cuts[1::2])]
        if trial % 3 == 0 and rs:  # empty runs are allowed
            rs.insert(1, rs[0] + rr[0]); rr.insert(1, 0)
        w = int(rng.integers(1, 400))
        lo = int(rng.integers(1, w + 1))
        run_model(16, rs, rr, n_rows, window_rows=w, min_direct_rows=lo, max_direct_rows=int(rng.integers(lo, 4 * w + 1)),
                  seed=trial)


def test_library_constants_on_a_sparse_byte_count():
    """The library's own window sizes for 256-byte rows, on run lengths of that scale (rows stand for themselves: one byte
    per row keeps the array small)."""
    window_rows, min_direct, max_direct = cm.library_windows(256)
    assert (window_rows, min_direct, max_direct) == (262144, 65536, 4194304)
    n_pages, page_rows = 4096, 1024
    keep = [p for p in range(n_pages) if (p // 16) % 10 >= 3]
    rs, rr = page_runs(keep, page_rows)
    windows = run_model(1, rs, rr, n_pages * page_rows, window_rows, min_direct, max_direct)
    # the 48 deleted pages in front displace the first window by 49152 rows, less than a direct window needs; after it
    # every window is direct
    assert [k for _, _, k in windows[:2]] == ["bounce", "direct"] and {k for _, _, k in windows[1:]} == {"direct"}
    assert sum(n for _, n, _ in windows) == len(keep) * page_rows


def test_bad_runs_are_refused_by_the_model():
    for rs, rr in (([0, 10], [20, 5]), ([10, 0], [5, 5]), ([0], [-1])):
        with pytest.raises(ValueError):
            cm.check_runs(rs, rr)


def test_new_entry_points_refuse_a_null_handle():
    from morphik_core_b200 import _native as nat

    out = ctypes.c_void_p()
    one = (ctypes.c_int64 * 1)(0)
    assert nat.lib.b200ms_block_create(None, 1 << 20, ctypes.byref(out)) == -1 and not out
    assert nat.lib.b200ms_block_create(None, -1, None) == -1
    assert nat.lib.b200ms_block_resize(None, None, 0) == -1
    assert nat.lib.b200ms_block_destroy(None, None) == -1
    assert nat.lib.b200ms_block_ptr(None) is None
    assert nat.lib.b200ms_block_mapped_bytes(None) == 0
    assert nat.lib.b200ms_compact_rows(None, None, 256, one, one, 1, None) == -1
