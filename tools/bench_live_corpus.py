"""Live-corpus probe (NOT the bench.py metric): what ingesting and compacting an HBM corpus costs in time and in device memory,
with the rows in a growable block (the product) and in torch buffers that grow by 1.5x with a copy and compact into a fresh
buffer (how the index worked before; kept callable here only, as OldIndex).  Both paths alternate in one process.  Prints the
card's name and power limit and one JSON line:

  ingest            the corpus added 256 pages per MaxSimIndex.add_pages call (what store_embeddings runs per call): wall
                    time, and the lowest free device memory seen after any call (torch.cuda.mem_get_info, synchronised)
  compact_documents after deleting 30 % of the documents (16 contiguous pages each);  compact_pages: after deleting 30 % of
                    the pages drawn singly (many short runs).  Wall time of the compact call around a synchronise and, for the
                    block, the device time of b200ms_compact_rows alone (CUDA events); bytes moved per second as a
                    fraction of a 4 GiB cudaMemcpyAsync device-to-device (bytes copied per second, measured in the same run);
                    free memory before and after the call, and torch's peak allocation during it
  largest_corpus    COMPUTED, not measured: the largest bf16 corpus that can be ingested 256 pages at a time and then survive
                    one compaction that keeps 70 %, from the peaks above and the free memory at the start.  The card is
                    shared: nothing here fills it or allocates until failure.

  python tools/bench_live_corpus.py [--pages 65536] [--reps 2]

--pages 65536 is 17.2 GB of bf16 rows; the old path needs up to 2.5x that while it grows, so the script refuses to start
with less than 3x free.
"""
import argparse
import ctypes
import json
import os
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

import numpy as np  # noqa: E402
import torch  # noqa: E402

import bench  # noqa: E402
from morphik_core_b200 import _native as nat  # noqa: E402
from morphik_core_b200.index import MaxSimIndex, _aligned_bytes, _padded_lens, _runs  # noqa: E402

ap = argparse.ArgumentParser()
ap.add_argument("--pages", type=int, default=65536)
ap.add_argument("--reps", type=int, default=2)
args = ap.parse_args()

DEV = torch.device("cuda", 0)
PAGE_ROWS, CALL_PAGES, ROW_BYTES = 1024, 256, 256
BOUNCE = 80 << 20  # b200ms_compact_rows' 64 MiB bounce buffer as the handle's scratch allocator rounds it


class OldIndex(MaxSimIndex):
    """The HBM index as it grew and compacted before the growable block: torch buffers, a copy per growth, a fresh buffer
    and one copy per run of surviving pages per compaction."""

    def _grow(self, need_rows, exact=False):
        if need_rows <= self._cap_rows:
            return
        new_cap = need_rows if exact else max(need_rows, int(self._cap_rows * 1.5), 4096)
        new_buf = _aligned_bytes(new_cap * self.row_bytes, self.device)
        if self._buf is not None and self._rows:
            new_buf[: self._rows * self.row_bytes].copy_(self._buf[: self._rows * self.row_bytes])
        self._buf, self._cap_rows, self._attached = new_buf, new_cap, False

    def compact(self, keep):
        pad = _padded_lens(self._page_lens)
        starts = np.concatenate([[0], np.cumsum(pad)]).astype(np.int64)
        new_rows = int(pad[keep].sum())
        new_buf = _aligned_bytes(max(new_rows, 4096) * self.row_bytes, self.device)
        dst = 0
        for first, last in _runs(keep):
            a, b = int(starts[first]) * self.row_bytes, int(starts[last + 1]) * self.row_bytes
            new_buf[dst:dst + (b - a)].copy_(self._buf[a:b])
            dst += b - a
        self._buf, self._cap_rows, self._rows = new_buf, new_buf.numel() // self.row_bytes, new_rows
        self._page_lens = [self._page_lens[p] for p in keep]
        self._attached = False


def free_bytes():
    torch.cuda.synchronize(DEV)
    return torch.cuda.mem_get_info(DEV)[0]


def settle():
    torch.cuda.synchronize(DEV)
    torch.cuda.empty_cache()
    torch.cuda.reset_peak_memory_stats(DEV)
    return free_bytes()


def ingest(cls, batch, n_pages):
    idx = cls(dtype="bf16")
    start = settle()
    lowest, t0 = start, time.perf_counter()
    for _ in range(n_pages // CALL_PAGES):
        idx.add_pages(batch)
        lowest = min(lowest, free_bytes())
    return idx, {"s": time.perf_counter() - t0, "lowest_free_gb": lowest / 1e9, "peak_used_gb": (start - lowest) / 1e9,
                 "torch_peak_gb": torch.cuda.max_memory_allocated(DEV) / 1e9}


def move_ms(idx, keep):
    """Device time (CUDA events) of b200ms_compact_rows alone on the index's rows, without the shrink that follows it in
    MaxSimIndex.compact.  It leaves the rows moved; the compaction timed after it moves the same runs again."""
    runs = [(a * PAGE_ROWS, (b + 1) * PAGE_ROWS) for a, b in _runs(keep)]
    run_start = np.array([a for a, _ in runs], dtype=np.int64)
    run_rows = np.array([b - a for a, b in runs], dtype=np.int64)
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    idx.h.check(nat.lib.b200ms_compact_rows(idx.h.ptr, ctypes.c_void_p(idx._buf.data_ptr()), ROW_BYTES,
                                            run_start.ctypes.data_as(nat.i64p), run_rows.ctypes.data_as(nat.i64p), len(runs),
                                            ctypes.c_void_p(torch.cuda.current_stream(DEV).cuda_stream)), "b200ms_compact_rows")
    e1.record()
    e1.synchronize()
    return e0.elapsed_time(e1)


def compact(idx, keep, copy_gbs):
    moved = len(keep) * PAGE_ROWS * ROW_BYTES
    out = {"runs": sum(1 for _ in _runs(keep)), "moved_gb": moved / 1e9}
    if not isinstance(idx, OldIndex):
        ms = move_ms(idx, keep)
        out.update({"move_ms": ms, "move_gbs": moved / 1e6 / ms, "move_fraction_of_memcpy": moved / 1e6 / ms / copy_gbs})
    start = settle()
    t0 = time.perf_counter()
    idx.compact(keep)
    after = free_bytes()
    s = time.perf_counter() - t0
    out.update({"s": s, "moved_gbs": moved / 1e9 / s, "fraction_of_memcpy": moved / 1e9 / s / copy_gbs,
                "free_before_gb": start / 1e9, "free_after_gb": after / 1e9,
                "torch_peak_gb": torch.cuda.max_memory_allocated(DEV) / 1e9})
    return out


def memcpy_gbs(nbytes=4 << 30):
    src = torch.empty(nbytes, dtype=torch.uint8, device=DEV)
    dst = torch.empty(nbytes, dtype=torch.uint8, device=DEV)
    best = 0.0
    for _ in range(4):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        dst.copy_(src, non_blocking=True)  # cudaMemcpyAsync device-to-device
        e1.record()
        e1.synchronize()
        best = max(best, nbytes / 1e9 / (e0.elapsed_time(e1) / 1e3))
    return best


def main():
    n_pages = args.pages // CALL_PAGES * CALL_PAGES
    corpus = n_pages * PAGE_ROWS * ROW_BYTES
    free0 = settle()
    if free0 < 3 * corpus:
        sys.exit(f"{free0 / 1e9:.1f} GB free, the old path's growth of a {corpus / 1e9:.1f} GB corpus needs up to 2.5x: "
                 f"pass a smaller --pages")
    print(f"[bench_live_corpus] {bench.gpu_name_and_power_limit(0)}; {free0 / 1e9:.1f} GB free at start", flush=True)
    g = torch.Generator(device=DEV)
    g.manual_seed(1)
    batch = torch.randn((CALL_PAGES * PAGE_ROWS, 128), generator=g, device=DEV)
    batch = list((batch / batch.norm(dim=1, keepdim=True)).to(torch.bfloat16).split(PAGE_ROWS))
    rng = np.random.default_rng(2)
    n_docs = n_pages // 16
    dead_docs = set(rng.choice(n_docs, size=int(0.3 * n_docs), replace=False).tolist())
    keeps = {"compact_documents": [p for p in range(n_pages) if p // 16 not in dead_docs],
             "compact_pages": np.flatnonzero(rng.random(n_pages) >= 0.3).tolist()}
    copy_gbs = memcpy_gbs()
    out = {"gpu": bench.gpu_name_and_power_limit(0), "pages": n_pages, "corpus_gb": corpus / 1e9, "free_at_start_gb": free0 / 1e9,
           "d2d_memcpy_gbs": copy_gbs, "reps": args.reps}
    runs = {"old": {"ingest": [], "compact_documents": [], "compact_pages": []},
            "new": {"ingest": [], "compact_documents": [], "compact_pages": []}}
    for _ in range(args.reps):
        for name, cls in (("old", OldIndex), ("new", MaxSimIndex)):
            for case, keep in keeps.items():
                idx, r = ingest(cls, batch, n_pages)
                runs[name]["ingest"].append(r)
                runs[name][case].append(compact(idx, keep, copy_gbs))
                idx.close()
                del idx
                settle()
    out["runs"] = runs
    # computed from free0, the free memory at the start.  New: what the ingest held beyond the corpus (a chunk, the pack
    # call's temporaries) plus the bounce buffer.  Old: torch's peak ALLOCATION (what it needs; its cache would be given
    # back under pressure) over ingest and compaction as a multiple of the corpus -- at this corpus size; where a size
    # falls in the 1.5x growth sequence moves the ingest peak between 1.67x and 2.5x.
    new_over = max(r["peak_used_gb"] for r in runs["new"]["ingest"]) * 1e9 - corpus + BOUNCE
    old_factor = max(r["torch_peak_gb"] for case in runs["old"].values() for r in case) * 1e9 / corpus
    out["largest_corpus_computed_gb"] = {"new": (free0 - new_over) / 1e9, "old": free0 / old_factor / 1e9,
                                         "old_worst_case": free0 / 2.5 / 1e9, "new_overhead_gb": new_over / 1e9,
                                         "old_factor": old_factor}
    print(json.dumps(out))


if __name__ == "__main__":
    main()
