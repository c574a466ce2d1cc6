"""The register plan of maxsim_wgmma_kernel, read from the built library (no GPU needed).

The producer warpgroup gives registers back with setmaxnreg.dec and the two consumer warpgroups take them with
setmaxnreg.inc, which waits until the CTA's register pool holds them.  The pool is what the launch allocated: 384 threads
at the kernel's register count.  So every instantiation must be compiled at 168 registers, and producer + 2 x consumer
must not exceed 3 x 168, or the kernel would hang on the GPU instead of failing here.
"""
import os
import re
import shutil
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LIB = os.path.join(ROOT, "morphik-core_b200", "lib", "libb200ms.so")
KERNEL = "maxsim_wgmma_kernel"
LAUNCH_REGS = 168  # 65536 registers / 384 threads, rounded down to a multiple of 8
# 1-bit corpus with 8 resident query tiles: the consumers need more than the 200 registers the 1-bit expander leaves them
SPILLS_ALLOWED = {"ILi1ELi8ELb1E"}


def _cuobjdump():
    for cand in (os.path.join(os.environ.get("CUDA_HOME", "/usr/local/cuda"), "bin", "cuobjdump"), shutil.which("cuobjdump")):
        if cand and os.path.exists(cand):
            return cand
    return None


@pytest.fixture(scope="module")
def dump():
    tool = _cuobjdump()
    if tool is None or not os.path.exists(LIB):
        pytest.skip("needs cuobjdump and the built libb200ms.so")

    def run(flag):
        return subprocess.run([tool, flag, LIB], capture_output=True, text=True, check=True).stdout

    return run("-res-usage"), run("-sass")


def _resources(res_usage):
    """{mangled kernel name: {REG: n, STACK: n, LOCAL: n}} of every maxsim_wgmma_kernel instantiation."""
    out, name = {}, None
    for line in res_usage.splitlines():
        m = re.search(r"Function (\S+):", line)
        if m:
            name = m.group(1)
            continue
        if name and KERNEL in name and "REG:" in line:
            out[name] = {k: int(v) for k, v in re.findall(r"(REG|STACK|LOCAL):(\d+)", line)}
            name = None
    return out


def _setmaxnreg(sass):
    """{mangled kernel name: (dealloc budgets, alloc budgets)} from the USETMAXREG instructions of each kernel."""
    out, name = {}, None
    for line in sass.splitlines():
        m = re.search(r"Function : (\S+)", line)
        if m:
            name = m.group(1)
            if KERNEL in name:
                out[name] = ([], [])
            continue
        if name in out:
            m = re.search(r"USETMAXREG\.(DEALLOC|TRY_ALLOC)\.CTAPOOL\s+(?:UP\d+,\s*)?(0x[0-9a-f]+)", line)
            if m:
                out[name][0 if m.group(1) == "DEALLOC" else 1].append(int(m.group(2), 16))
    return out


def test_every_instantiation_runs_at_the_launch_register_count(dump):
    res = _resources(dump[0])
    assert len(res) == 14, sorted(res)
    for name, r in res.items():
        assert r["REG"] == LAUNCH_REGS, (name, r)


def test_no_local_memory(dump):
    for name, r in _resources(dump[0]).items():
        assert r["LOCAL"] == 0, (name, r)
        if not any(tag in name for tag in SPILLS_ALLOWED):
            assert r["STACK"] == 0, (name, r)


def test_register_budgets_fit_the_pool(dump):
    plans = _setmaxnreg(dump[1])
    assert len(plans) == 14, sorted(plans)
    for name, (dec, inc) in plans.items():
        assert len(dec) == 1 and len(inc) == 1, (name, dec, inc)  # producer gives back once, consumers take once
        assert dec[0] + 2 * inc[0] <= 3 * LAUNCH_REGS, (name, dec, inc)
        if "ELb0E" in name and ("ILi0E" in name or "ILi1E" in name):  # TMA producers: one thread issues the loads
            assert (dec[0], inc[0]) == (40, 232), (name, dec, inc)
