"""ctypes binding of libb200ms.so -- the only way the Python host reaches the GPU kernels.

The declarations mirror include/b200ms.h one to one (tests/test_cabi_symbols.py checks that every symbol the
header declares is exported).  Importing this module never touches CUDA; creating a handle does and raises
``NativeError`` when no H100 is present.  There is deliberately no fallback implementation.
"""
from __future__ import annotations

import ctypes
import os
from ctypes import POINTER, c_char_p, c_float, c_int, c_int32, c_int64, c_void_p

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "lib", "libb200ms.so")

F32, BF16, I8, B1, I32, F8 = 0, 1, 2, 3, 4, 5
DTYPE_NAMES = {"f32": F32, "bf16": BF16, "int8": I8, "i8": I8, "binary": B1, "b1": B1, "1bit": B1, "fp8": F8, "f8": F8,
               "e4m3": F8}
ROW_BYTES = {F32: 512, BF16: 256, I8: 128, B1: 16, F8: 128}
DIM = 128
ROW_GROUP = 32
MAX_K = 4096


class NativeError(RuntimeError):
    """A libb200ms call failed (the message is b200ms_last_error)."""


def _load() -> ctypes.CDLL:
    override = os.environ.get("B200MS_LIB")  # developer A/B aid: an explicit variant of the library
    if override:
        return _declare(ctypes.CDLL(override))
    if not os.path.exists(LIB_PATH):
        raise ImportError(
            f"{LIB_PATH} is missing: build it with `python __graft_entry__.py build` "
            "(nvcc, sm_90a). morphik-core_b200 has no CPU fallback."
        )
    from . import build_native

    if build_native.mismatched():  # a library built from older sources would silently run old kernels
        raise ImportError(
            f"{LIB_PATH} does not match morphik-core_b200/csrc (source hash differs): rebuild it with "
            "`python __graft_entry__.py build`."
        )
    return _declare(ctypes.CDLL(LIB_PATH))


# (restype, argtypes) of every function include/b200ms.h declares
vp, i32p, i64p, f32p = c_void_p, POINTER(c_int32), POINTER(c_int64), POINTER(c_float)
_SIGNATURES = {
    "b200ms_version": (c_int, []),
    "b200ms_device_count": (c_int, []),
    "b200ms_create": (c_int, [c_int, POINTER(c_void_p)]),
    "b200ms_destroy": (c_int, [vp]),
    "b200ms_last_error": (c_char_p, [vp]),
    "b200ms_padded_len": (c_int64, [c_int64]),
    "b200ms_padded_rows": (c_int64, [i32p, c_int64]),
    "b200ms_row_bytes": (c_int64, [c_int]),
    "b200ms_query_groups": (c_int64, [i32p, c_int]),
    "b200ms_sign_pack": (c_int, [vp, vp, c_int, c_int64, vp, vp]),
    "b200ms_hamming_batch": (c_int, [vp, vp, vp, c_int64, vp, vp]),
    "b200ms_pack_pages": (c_int, [vp, vp, c_int, i32p, c_int64, vp, c_int, c_float, vp]),
    "b200ms_set_corpus": (c_int, [vp, vp, c_int, i32p, c_int64]),
    "b200ms_corpus_pages": (c_int64, [vp]),
    "b200ms_corpus_rows": (c_int64, [vp]),
    "b200ms_pack_queries": (c_int, [vp, vp, c_int, i32p, c_int, vp, c_int, c_float, i32p, POINTER(c_int), vp]),
    "b200ms_score": (c_int, [vp, vp, c_int, i32p, i32p, c_int, vp, c_int64, vp]),
    "b200ms_topk": (c_int, [vp, vp, c_int, c_int64, c_int64, i32p, c_int, vp, c_int, c_float, c_int64, vp, vp, vp, vp]),
    "b200ms_topk_masked": (c_int, [vp, vp, c_int, c_int64, c_int64, i32p, c_int, vp, c_int, vp, c_int, c_float, c_int64, vp, vp,
                                   vp, vp]),
    "b200ms_merge_topk": (c_int, [vp, vp, vp, c_int, c_int, c_int, vp, vp, vp, vp]),
    "b200ms_search_host": (c_int, [vp, vp, i32p, c_int, c_int, vp, c_float, c_float, c_int64, vp, vp, vp]),
    "b200ms_search_host_masked": (c_int, [vp, vp, i32p, c_int, c_int, vp, c_int, i32p, c_float, c_float, c_int64, vp, vp, vp]),
    "b200ms_search_device": (c_int, [vp, vp, c_int, i32p, c_int, c_int, vp, c_float, c_float, c_int64, vp, vp, vp, vp]),
    "b200ms_search_device_masked": (c_int, [vp, vp, c_int, i32p, c_int, c_int, vp, c_int, vp, c_float, c_float, c_int64, vp, vp,
                                    vp, vp]),
    "b200ms_launch_count": (c_int64, [vp]),
    "b200ms_last_score_ms": (c_float, [vp]),
    "b200ms_set_tuning": (c_int, [vp, c_int64, c_int]),
    "b200ms_set_option": (c_int, [vp, c_char_p, c_int64]),
    "b200ms_rerank_device": (c_int, [vp, vp, c_int, i32p, c_int, vp, c_int, c_int, c_float, c_float, vp, vp, vp, vp]),
    "b200ms_rerank_batch_device": (c_int, [vp, vp, c_int, i32p, c_int, vp, c_int, c_int, c_float, c_float, vp, vp, vp, vp]),
    "b200ms_comm_available": (c_int, []),
    "b200ms_comm_unique_id": (c_int, [vp]),
    "b200ms_comm_init": (c_int, [vp, vp, c_int, c_int]),
    "b200ms_comm_adopt": (c_int, [vp, vp, c_int, c_int]),
    "b200ms_comm_destroy": (c_int, [vp]),
    "b200ms_comm_rank": (c_int, [vp]),
    "b200ms_comm_world": (c_int, [vp]),
    "b200ms_xchg_bytes": (c_int64, [c_int, c_int]),
    "b200ms_bcast_device": (c_int, [vp, vp, c_int64, c_int, vp]),
    "b200ms_allgather_topk": (c_int, [vp, vp, vp, c_int, c_int, vp, vp, vp, vp]),
    "b200ms_send_device": (c_int, [vp, vp, c_int64, c_int, vp]),
    "b200ms_recv_device": (c_int, [vp, vp, c_int64, c_int, vp]),
    "b200ms_sharded_search_begin": (c_int64, [vp, vp, c_int, i32p, c_int, c_int, vp, c_int, vp, c_float, c_float, c_int64, vp,
                                    vp, vp, vp]),
    "b200ms_sharded_search_end": (c_int, [vp, c_int64, vp]),
    "b200ms_sharded_search_host_begin": (c_int64, [vp, vp, i32p, c_int, c_int, vp, c_int, vp, c_float, c_float, c_int64]),
    "b200ms_sharded_search_host_end": (c_int, [vp, c_int64, vp, vp, vp]),
    "b200ms_fde_configure_ex": (c_int, [vp, c_int, c_int, c_int, c_float, vp, vp, vp, c_int, c_int, vp, vp]),
    "b200ms_fde_configure": (c_int, [vp, c_int, c_int, c_int, c_float, vp, vp, vp]),
    "b200ms_fde_dim": (c_int64, [vp]),
    "b200ms_fde_encode": (c_int, [vp, vp, c_int, i32p, c_int64, c_int, vp, vp]),
    "b200ms_fde_finalize": (c_int, [vp, vp, c_int64, vp, vp, vp]),
    "b200ms_fde_encode_corpus": (c_int, [vp, c_int64, c_int64, vp, vp]),
    "b200ms_fde_scan": (c_int, [vp, vp, vp, c_int64, vp, c_int, vp, c_int64, vp]),
    "b200ms_score_call_count": (c_int64, [vp]),
    "b200ms_score_times_ms": (c_int, [vp, f32p, c_int]),
    "b200ms_set_corpus_host": (c_int, [vp, vp, c_int, i32p, c_int64]),
    "b200ms_host_alloc": (c_int, [vp, c_int64, POINTER(c_void_p)]),
    "b200ms_host_free": (c_int, [vp, vp]),
    "b200ms_last_gather_stats": (c_int, [vp, i64p, i64p, POINTER(c_int), f32p]),
    "b200ms_block_create": (c_int, [vp, c_int64, POINTER(c_void_p)]),
    "b200ms_block_resize": (c_int, [vp, vp, c_int64]),
    "b200ms_block_ptr": (c_void_p, [vp]),
    "b200ms_block_mapped_bytes": (c_int64, [vp]),
    "b200ms_block_destroy": (c_int, [vp, vp]),
    "b200ms_compact_rows": (c_int, [vp, vp, c_int64, i64p, i64p, c_int64, vp]),
    "b200ms_last_scan_stats": (c_int, [vp, i64p, i64p]),
    "b200ms_explain_device": (c_int, [vp, vp, c_int, i32p, c_int, vp, c_int, c_float, c_float, vp, vp, vp, c_int64, vp]),
    "b200ms_topk_docs": (c_int, [vp, vp, c_int, c_int64, c_int64, i32p, c_int, vp, vp, c_int64, c_int, c_int, c_float, c_int64,
                                 vp, vp, vp, vp, vp]),
    "b200ms_search_docs_device": (c_int, [vp, vp, c_int, i32p, c_int, c_int, c_int, vp, c_int64, vp, c_int, vp, c_float, c_float,
                                          c_int64, vp, vp, vp, vp, vp]),
    "b200ms_rerank_docs_batch_device": (c_int, [vp, vp, c_int, i32p, c_int, vp, c_int, c_int, c_int, vp, c_int64, c_float,
                                                c_float, vp, vp, vp, vp, vp]),
    "b200ms_sign_rows": (c_int, [vp, c_int64, c_int64, vp, vp]),
    "b200ms_set_sign_rows": (c_int, [vp, vp, c_int64, vp]),
    "b200ms_sign_candidates_device": (c_int, [vp, vp, c_int, i32p, c_int, c_int, vp, c_int, vp, c_float, c_float, vp, vp, vp,
                                              vp]),
    "b200ms_mmr_device": (c_int, [vp, vp, vp, c_int, i32p, c_int, c_int, c_float, c_float, vp, vp, vp, vp, vp]),
    "b200ms_search_pages_device": (c_int, [vp, i64p, c_int, c_int, vp, c_int, vp, c_float, c_int64, vp, vp, vp, vp]),
    "b200ms_rerank_pages_batch_device": (c_int, [vp, i64p, c_int, vp, c_int, c_int, vp, c_int, vp, c_float, vp, vp, vp, vp]),
    "b200ms_page_rows_device": (c_int, [vp, i64p, c_int, c_float, vp, vp]),
    "b200ms_search_examples_device": (c_int, [vp, vp, c_int, i32p, c_int, i64p, c_int, i32p, f32p, c_int, c_int, vp, c_int, vp,
                                              c_float, c_float, c_int64, vp, vp, vp, vp]),
    "b200ms_rerank_examples_batch_device": (c_int, [vp, vp, c_int, i32p, c_int, i64p, c_int, i32p, f32p, c_int, vp, c_int, c_int,
                                                    vp, c_int, vp, c_float, c_float, vp, vp, vp, vp]),
    "b200ms_union_candidates_device": (c_int, [vp, vp, c_int, c_int, i32p, c_int, vp, c_int, vp]),
    "b200ms_search_doc_maxsim_device": (c_int, [vp, vp, c_int, i32p, c_int, c_int, c_int, vp, c_int64, vp, c_int, vp, c_float,
                                                c_float, c_int64, vp, vp, vp, vp, vp, vp, vp]),
    "b200ms_rerank_doc_maxsim_batch_device": (c_int, [vp, vp, c_int, i32p, c_int, vp, c_int, c_int, c_int, vp, c_int64, vp,
                                                      c_int, vp, c_float, c_float, c_int64, vp, vp, vp, vp, vp, vp, vp]),
    "b200ms_pair_maxsim_device": (c_int, [vp, vp, vp, c_int64, c_float, vp, vp, vp]),
    "b200ms_duplicate_groups_device": (c_int, [vp, vp, vp, vp, vp, c_int64, c_float, vp, vp, vp]),
}


def _declare(lib: ctypes.CDLL) -> ctypes.CDLL:
    for name, (res, args) in _SIGNATURES.items():
        fn = getattr(lib, name)
        fn.restype = res
        fn.argtypes = args
    return lib


lib = _load()
EXPORTED = list(_SIGNATURES)
MAX_PER_DOC = 64


def i32_array(values):
    arr = (c_int32 * len(values))(*[int(v) for v in values])
    return arr


def i64_array(values):
    return (c_int64 * len(values))(*[int(v) for v in values])


def f32_array(values):
    return (c_float * len(values))(*[float(v) for v in values])


class Handle:
    """RAII wrapper of b200ms_t*; ``check`` turns error codes into NativeError."""

    def __init__(self, device: int = 0):
        self._h = c_void_p()
        rc = lib.b200ms_create(int(device), ctypes.byref(self._h))
        if rc != 0:
            msg = lib.b200ms_last_error(None)
            raise NativeError(f"b200ms_create(device={device}) failed ({rc}): {msg.decode() if msg else ''}")
        self.device = int(device)

    @property
    def ptr(self):
        return self._h

    def check(self, rc: int, what: str = ""):
        if rc != 0:
            msg = lib.b200ms_last_error(self._h)
            raise NativeError(f"{what or 'libb200ms'} failed ({rc}): {msg.decode() if msg else ''}")

    def close(self):
        if self._h:
            lib.b200ms_destroy(self._h)
            self._h = c_void_p()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass
