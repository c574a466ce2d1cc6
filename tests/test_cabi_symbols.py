"""CPU checks of the drop-in boundary: libb200ms.so loads, exports every symbol include/b200ms.h declares, the pure
host helpers compute the documented layout arithmetic, and compute entry points FAIL LOUDLY without a GPU
(no CPU fallback anywhere in the product path)."""
import ctypes
import os
import re
import subprocess

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def header_symbols():
    text = open(os.path.join(ROOT, "include", "b200ms.h")).read()
    text = re.sub(r"/\*.*?\*/", "", text, flags=re.S)
    return sorted(set(re.findall(r"\b(b200ms_[a-z0-9_]+)\s*\(", text)))


def test_header_symbols_all_exported_and_bound():
    from morphik_core_b200 import _native as nat

    syms = header_symbols()
    assert len(syms) >= 20
    out = subprocess.run(["nm", "-D", "--defined-only", nat.LIB_PATH], capture_output=True, text=True, check=True).stdout
    exported = set(re.findall(r" T (b200ms_[a-z0-9_]+)", out))
    assert set(syms) == exported, (sorted(set(syms) - exported), sorted(exported - set(syms)))
    assert sorted(nat.EXPORTED) == syms  # the ctypes binding covers the whole header
    for s in syms:
        assert getattr(nat.lib, s).argtypes is not None


def test_no_oracle_or_cpu_fallback_in_product_path():
    pkg = os.path.join(ROOT, "morphik-core_b200")
    for dirpath, _, files in os.walk(pkg):
        for f in files:
            if f.endswith((".py", ".cu", ".cuh", ".h")):
                src = open(os.path.join(dirpath, f)).read()
                assert "from oracle" not in src and "import oracle" not in src and "maxsim_oracle" not in src, f
    out = subprocess.run(["ldd", os.path.join(pkg, "lib", "libb200ms.so")], capture_output=True, text=True).stdout
    assert "liboracle" not in out


def test_layout_helpers():
    from morphik_core_b200 import _native as nat

    lib = nat.lib
    assert lib.b200ms_version() == 200
    assert [lib.b200ms_padded_len(n) for n in (0, 1, 31, 32, 33, 1024, 1030)] == [0, 32, 32, 32, 64, 1024, 1056]
    lens = nat.i32_array([0, 1, 32, 33, 1024])
    assert lib.b200ms_padded_rows(lens, 5) == 0 + 32 + 32 + 64 + 1024
    assert [lib.b200ms_row_bytes(d) for d in (nat.F32, nat.BF16, nat.I8, nat.B1, nat.F8, 99)] == [512, 256, 128, 16, 128, 0]
    assert lib.b200ms_query_groups(nat.i32_array([32, 20, 33, 0, 1030]), 5) == 1 + 1 + 2 + 0 + 33


def test_fails_loudly_without_gpu():
    import torch

    from morphik_core_b200 import _native as nat

    if torch.cuda.is_available():
        pytest.skip("this check is for the CPU-only build container")
    assert nat.lib.b200ms_device_count() == 0
    with pytest.raises(nat.NativeError, match="no CUDA device"):
        nat.Handle(0)
    from morphik_core_b200.index import MaxSimIndex

    with pytest.raises(nat.NativeError):
        MaxSimIndex(dtype="bf16")
    from morphik_core_b200.store import B200MultiVectorStore

    with pytest.raises(nat.NativeError):
        B200MultiVectorStore(mode="bf16")  # auto_initialize -> needs the GPU; nothing to fall back to
    # NULL handle -> EINVAL, never a crash
    assert nat.lib.b200ms_set_corpus(None, None, nat.BF16, None, 0) == -1


def test_sass_has_hopper_tensor_and_tma_instructions():
    """Static evidence that the hot kernels are sm_90a warpgroup-MMA + TMA code: bf16, int8 and f16 (the widened e4m3 corpora) wgmma,
    TMA loads."""
    from morphik_core_b200 import _native as nat

    cuobjdump = "/usr/local/cuda/bin/cuobjdump"
    if not os.path.exists(cuobjdump):
        pytest.skip("cuobjdump not available")
    sass = subprocess.run([cuobjdump, "-sass", nat.LIB_PATH], capture_output=True, text=True).stdout
    for mnemonic in ("HGMMA.64x128x16.F32.BF16", "IGMMA.64x128x32.S8.S8", "HGMMA.64x128x16.F32 ", "HGMMA.64x64x16",
                     "UTMALDG", "POPC"):
        assert mnemonic in sass, mnemonic
    assert "HMMA.16816" not in sass  # no legacy mma.sync path


def test_library_matches_sources_and_stale_library_is_detected(tmp_path, monkeypatch):
    """libb200ms.so carries a stamp of the sources it was built from; a mismatch must be detected (the loader then refuses
    the library instead of silently running kernels from older sources)."""
    from morphik_core_b200 import build_native as bn

    assert os.path.exists(bn.STAMP) and not bn.stale() and not bn.mismatched()
    fake = tmp_path / "libb200ms.so.srchash"
    fake.write_text("0" * 64 + "\n")
    monkeypatch.setattr(bn, "STAMP", str(fake))
    assert bn.stale() and bn.mismatched()
    monkeypatch.setattr(bn, "STAMP", str(tmp_path / "absent"))
    assert bn.stale() and not bn.mismatched()  # no stamp: rebuild wanted, but the library cannot be called wrong


def test_every_named_option_is_documented_in_the_header():
    """b200ms_set_option names (csrc/api.cu) <-> the option list in include/b200ms.h: a knob without documentation is invisible
    to a ctypes-only host."""
    import re

    api = open(os.path.join(ROOT, "morphik-core_b200", "csrc", "api.cu")).read()
    body = api[api.index("B200MS_API int b200ms_set_option"):]
    body = body[:body.index("\n}\n")]
    names = set(re.findall(r'n == "([a-z0-9_]+)"', body))
    assert {"b1_tensor", "fde_gemm", "zero_pad_compat"} <= names
    header = open(os.path.join(ROOT, "include", "b200ms.h")).read()
    missing = sorted(n for n in names if f'"{n}"' not in header)
    assert not missing, f"options without a line in include/b200ms.h: {missing}"
