"""Build libb200ms.so (the C-ABI CUDA library) in-tree with nvcc for sm_90a (H100).

Usage: python morphik-core_b200/build_native.py [--force]
The output morphik-core_b200/lib/libb200ms.so (and the objects, build.log and source stamp beside it) is git-ignored.
"""
import os
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
LIB_DIR = os.path.join(HERE, "lib")
LIB = os.path.join(LIB_DIR, "libb200ms.so")
SOURCES = ["api.cu", "maxsim_wgmma.cu", "maxsim_b1.cu", "pack.cu", "topk.cu", "fde.cu", "comm.cu", "host_tier.cu", "maxsim_explain.cu",
           "topk_docs.cu", "scan_plan.cu", "block.cu", "compact.cu", "signs.cu", "maxsim_mmr.cu",
           "search_pages.cu", "search_examples.cu", "doc_maxsim.cu", "duplicates.cu"]
HEADERS = ["common.cuh", "ptx.cuh", "mma_tile.cuh", "topk_keys.cuh", "scan.cuh", "row_tiles.cuh", os.path.join("..", "..", "include", "b200ms.h")]
NVCC_FLAGS = [
    "-gencode", "arch=compute_90a,code=sm_90a", "-lineinfo", "-O3", "-std=c++17",
    "-Xcompiler", "-fPIC,-fvisibility=hidden", "-Xptxas", "-v", "--expt-relaxed-constexpr",
]


def _nvcc() -> str:
    for cand in (os.environ.get("NVCC"), "/usr/local/cuda/bin/nvcc", "nvcc"):
        if cand and (os.path.isabs(cand) and os.path.exists(cand) or not os.path.isabs(cand)):
            return cand
    return "nvcc"


STAMP = LIB + ".srchash"


def source_hash() -> str:
    """sha256 over the CUDA sources, headers and compiler flags: the identity of what libb200ms.so was built from."""
    import hashlib

    h = hashlib.sha256(" ".join(NVCC_FLAGS).encode())
    for rel in SOURCES + HEADERS:
        h.update(rel.encode())
        with open(os.path.join(CSRC, rel), "rb") as f:
            h.update(f.read())
    return h.hexdigest()


def stale() -> bool:
    """True when the library is missing or was built from different sources (content hash, so it also works on a copy of
    the tree whose mtimes are meaningless)."""
    if not (os.path.exists(LIB) and os.path.exists(STAMP)):
        return True
    with open(STAMP) as f:
        return f.read().strip() != source_hash()


def mismatched() -> bool:
    """True only when a stamp exists and names different sources (a library without a stamp cannot be judged)."""
    if not (os.path.exists(LIB) and os.path.exists(STAMP)):
        return False
    with open(STAMP) as f:
        return f.read().strip() != source_hash()


def build(force: bool = False, verbose: bool = False) -> str:
    if not (force or stale()):
        return LIB
    os.makedirs(LIB_DIR, exist_ok=True)
    objs = []
    procs = []
    for src in SOURCES:
        obj = os.path.join(LIB_DIR, src.replace(".cu", ".o"))
        cmd = [_nvcc()] + NVCC_FLAGS + ["-c", os.path.join(CSRC, src), "-o", obj]
        procs.append((src, subprocess.Popen(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)))
        objs.append(obj)
    log = []
    failed = False
    for src, p in procs:
        out, _ = p.communicate()
        log.append(f"==== {src}\n{out}")
        failed |= p.returncode != 0
    with open(os.path.join(LIB_DIR, "build.log"), "w") as f:
        f.write("\n".join(log))
    if failed or verbose:
        print("\n".join(log))
    if failed:
        raise RuntimeError("nvcc failed; see output above")
    link = [_nvcc(), "-shared", "-gencode", "arch=compute_90a,code=sm_90a", "-o", LIB] + objs + ["-ldl"]
    subprocess.run(link, check=True)
    with open(STAMP, "w") as f:
        f.write(source_hash() + "\n")
    return LIB


if __name__ == "__main__":
    print(build(force="--force" in sys.argv, verbose=True))
