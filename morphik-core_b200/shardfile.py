"""Packed shard files -- the durable form of a device corpus (SURVEY 8f-2).

The reference keeps multivectors as one object per page: ``numpy.save`` of float32 ``[P,128]`` under
``multivector/{document_id}/{chunk_number}.npy`` (core/vector_store/fast_multivector_store.py:673-707, read back one by one
at :713-774 through a disk LRU cache), or as ``BIT(128)[]`` rows in Postgres (multi_vector_store.py:240-251).  Rebuilding a
GPU corpus from those costs one object fetch / row decode per page.  A shard file is the packed HBM layout itself,
so loading is a sequence of large sequential reads + H2D copies and nothing else:

    offset 0     : 4096-byte header  = magic "B2MSHARD", version, dtype, n_pages, n_rows_padded, row_bytes, i8_scale (JSON, NUL padded)
    offset 4096  : page_lens  int32[n_pages]   (true lengths), zero padded to a 4096-byte boundary
    then         : rows       n_rows_padded * row_bytes bytes, exactly as they sit in HBM

Importers for the reference's durable forms: ``import_npy_pages`` (float32 .npy files) and ``pages_from_bit_rows``
(packed 16-byte sign-bit rows as pgvector's ``Bit`` stores them, multi_vector_store.py:339-345).
"""
from __future__ import annotations

import json
import os
from typing import Iterable, List, Optional, Sequence, Tuple

import numpy as np
import torch

from . import _native as nat
from .index import MaxSimIndex

MAGIC = "B2MSHARD"
HEADER_BYTES = 4096
CHUNK_BYTES = 256 << 20  # staging granularity for file <-> pinned <-> device copies


def _round_up(x: int, a: int) -> int:
    return (x + a - 1) // a * a


def save_index(index: MaxSimIndex, path: str, first_page: int = 0, n_pages: Optional[int] = None) -> int:
    """Write the packed corpus of `index` (or only pages [first_page, first_page + n_pages): a journal segment) to `path`;
    returns bytes written."""
    all_lens = np.asarray(index.page_lens, dtype=np.int32)
    n_pages = len(all_lens) - first_page if n_pages is None else int(n_pages)
    lens = all_lens[first_page:first_page + n_pages]
    r0, r1 = index.page_row_range(first_page, n_pages)
    rows = index.packed_rows()[r0:r1].reshape(-1)  # uint8 device view
    header = {"magic": MAGIC, "version": 1, "dtype": index.dtype_name, "n_pages": int(len(lens)),
              "n_rows_padded": int(r1 - r0), "row_bytes": int(index.row_bytes), "i8_scale": float(index.i8_scale)}
    blob = json.dumps(header).encode()
    assert len(blob) < HEADER_BYTES
    lens_bytes = _round_up(lens.nbytes, 4096)
    with open(path, "wb") as f:
        f.write(blob.ljust(HEADER_BYTES, b"\0"))
        f.write(lens.tobytes().ljust(lens_bytes, b"\0"))
        total = rows.numel()
        stage = torch.empty(min(CHUNK_BYTES, max(total, 1)), dtype=torch.uint8).pin_memory()
        for o in range(0, total, CHUNK_BYTES):
            n = min(CHUNK_BYTES, total - o)
            stage[:n].copy_(rows[o:o + n])  # D2H into pinned memory (synchronous for a pinned destination)
            f.write(stage[:n].numpy().tobytes() if n < stage.numel() else stage.numpy().data)
    return HEADER_BYTES + lens_bytes + int(rows.numel())


def read_header(path: str) -> Tuple[dict, np.ndarray, int]:
    with open(path, "rb") as f:
        raw = f.read(HEADER_BYTES)
        header = json.loads(raw.rstrip(b"\0").decode())
        if header.get("magic") != MAGIC or header.get("version") != 1:
            raise ValueError(f"{path}: not a B2MSHARD v1 file")
        lens = np.frombuffer(f.read(4 * header["n_pages"]), dtype=np.int32).copy()
    payload_off = HEADER_BYTES + _round_up(4 * header["n_pages"], 4096)
    return header, lens, payload_off


def load_index(path: str, device: int = 0, into: Optional[MaxSimIndex] = None, tier: str = "hbm") -> MaxSimIndex:
    """Read a shard file into the index's own block (no repacking, no second copy of the corpus): a new index of the file's
    dtype on tier `tier`, or with ``into`` an existing index of the same dtype that the pages are APPENDED to (journal
    segments).  Host-tier rows are read straight into the pinned block; device rows go through two pinned staging buffers."""
    header, lens, payload_off = read_header(path)
    if into is not None and (into.dtype_name != header["dtype"] or float(into.i8_scale) != float(header["i8_scale"])):
        raise ValueError(f"{path}: segment dtype/scale differs from the index it is appended to")
    index = into if into is not None else MaxSimIndex(device=device, dtype=header["dtype"], i8_scale=header["i8_scale"],
                                                      tier=tier)
    total = header["n_rows_padded"] * header["row_bytes"]
    if int(nat.lib.b200ms_padded_rows(nat.i32_array(lens.tolist()), len(lens))) != header["n_rows_padded"]:
        raise ValueError(f"{path}: page lengths do not match the row count")
    if os.path.getsize(path) < payload_off + total:
        raise ValueError(f"{path}: truncated payload")
    index.reserve_rows(index.n_rows_padded + header["n_rows_padded"])
    dst = index.tail(total)
    staged = dst.is_cuda  # double-buffered: chunk i+1 is read into one staging buffer while chunk i copies from the other
    stages = [torch.empty(min(CHUNK_BYTES, max(total, 1)), dtype=torch.uint8).pin_memory()
              for _ in range(2 if staged else 0)]
    events = [torch.cuda.Event(), torch.cuda.Event()]
    with open(path, "rb") as f, torch.cuda.device(index.device):
        f.seek(payload_off)
        for i, o in enumerate(range(0, total, CHUNK_BYTES)):
            n = min(CHUNK_BYTES, total - o)
            if staged and i >= 2:
                events[i & 1].synchronize()
            target = stages[i & 1][:n] if staged else dst[o:o + n]
            if f.readinto(memoryview(target.numpy())) != n:
                raise ValueError(f"{path}: short read")
            if staged:
                dst[o:o + n].copy_(target, non_blocking=True)
                events[i & 1].record()
        torch.cuda.current_stream().synchronize()
    index.commit_rows(lens.tolist())
    return index


class StoreJournal:
    """Append-only durable form of a store directory (SURVEY 8f-2 "incremental append/delete by document").

    The reference persists every ``store_embeddings`` call as it happens (one ``.npy`` per page,
    fast_multivector_store.py:673-707; rows in Postgres, multi_vector_store.py:681-703) and deletes by document id
    (multi_vector_store.py:929-933).  Here the same two operations append to a directory instead of rewriting one file:

        journal.log          one JSON line per operation, in order:
                               {"op":"segment","seq":N,"pages":P}      pages added by one store_embeddings call
                               {"op":"delete","document_id":"..."}     tombstone
        seg-NNNNNN.b2ms      the packed rows of those pages (B2MSHARD v1, exactly the HBM layout)
        seg-NNNNNN.cat.jsonl their catalogue records (document_id, chunk_number, content, metadata, app_id, n_rows)
        seg-NNNNNN.fde.pt    (two-stage stores) their FDE rows + inverse norms

    Replaying the log in order reproduces the store; ``checkpoint`` (store.save) rewrites the live pages as one segment and
    truncates the log.  Every file is written to a temporary name and renamed, the log line is appended (and fsynced) last,
    so a crash leaves either the old state or the new one.
    """

    LOG = "journal.log"

    def __init__(self, directory: str):
        self.dir = directory
        os.makedirs(directory, exist_ok=True)
        self.seq = 0
        for op in self.read_ops():
            if op.get("op") == "segment":
                self.seq = max(self.seq, int(op["seq"]))

    def _path(self, name: str) -> str:
        return os.path.join(self.dir, name)

    def read_ops(self) -> List[dict]:
        p = self._path(self.LOG)
        if not os.path.exists(p):
            return []
        ops = []
        with open(p) as f:
            for line in f:
                line = line.strip()
                if not line:
                    continue
                try:
                    ops.append(json.loads(line))
                except json.JSONDecodeError:  # a torn last line (crash mid-append): everything before it is intact
                    break
        return ops

    def _append(self, op: dict) -> None:
        with open(self._path(self.LOG), "a") as f:
            f.write(json.dumps(op) + "\n")
            f.flush()
            os.fsync(f.fileno())

    def log_add(self, index: MaxSimIndex, first_page: int, n_pages: int, records: Sequence[dict], fde=None) -> int:
        self.seq += 1
        stem = f"seg-{self.seq:06d}"
        tmp = self._path(stem + ".b2ms.tmp")
        save_index(index, tmp, first_page, n_pages)
        os.replace(tmp, self._path(stem + ".b2ms"))
        tmp = self._path(stem + ".cat.jsonl.tmp")
        with open(tmp, "w") as f:
            for r in records:
                f.write(json.dumps(r) + "\n")
        os.replace(tmp, self._path(stem + ".cat.jsonl"))
        if fde is not None:
            rows, inv = fde
            tmp = self._path(stem + ".fde.pt.tmp")
            torch.save({"rows": rows.detach().cpu().view(torch.int16), "inv": inv.detach().cpu()}, tmp)
            os.replace(tmp, self._path(stem + ".fde.pt"))
        self._append({"op": "segment", "seq": self.seq, "pages": int(n_pages)})
        return self.seq

    def log_delete(self, document_id: str) -> None:
        self._append({"op": "delete", "document_id": document_id})

    def segment_files(self, seq: int) -> Tuple[str, str, str]:
        stem = f"seg-{int(seq):06d}"
        return self._path(stem + ".b2ms"), self._path(stem + ".cat.jsonl"), self._path(stem + ".fde.pt")

    def reset(self) -> None:
        """Drop every segment and the log (checkpoint writes a fresh base segment right after)."""
        for name in os.listdir(self.dir):
            if name == self.LOG or name.startswith("seg-"):
                os.remove(self._path(name))
        self.seq = 0


def import_npy_pages(index: MaxSimIndex, paths: Sequence[str], batch: int = 256) -> int:
    """Append pages stored the reference's way (one float32 [P,128] ``.npy`` per page, fast_multivector_store.py:673-707)."""
    n = 0
    for i in range(0, len(paths), batch):
        pages = [np.load(p).astype(np.float32, copy=False).reshape(-1, nat.DIM) for p in paths[i:i + batch]]
        index.add_pages(pages)
        n += len(pages)
    return n


def pages_from_bit_rows(rows_per_page: Iterable[Sequence[bytes]]) -> List[np.ndarray]:
    """Postgres ``BIT(128)[]`` rows (each element the 16 packed bytes pgvector's ``Bit`` holds, MSB first) -> float32 +-1
    pages whose sign bits are exactly those bits -- feed to a ``dtype="binary"`` index (sign(x) > 0 recovers every bit; this
    is the migration path of scripts/migrate_postgres_to_turbopuffer.py:233-273 in the other direction)."""
    pages = []
    for rows in rows_per_page:
        arr = np.frombuffer(b"".join(rows), dtype=np.uint8).reshape(-1, 16) if len(rows) else np.zeros((0, 16), np.uint8)
        bits = np.unpackbits(arr, axis=1, bitorder="big").astype(np.float32)
        pages.append(bits * 2.0 - 1.0)
    return pages
