"""The block-diagonal solver's packed bookkeeping (`Bookkeeping<true>` in dexr_kernels.cuh: two 32-bit words) must read back
what the dense and arrow solvers' unpacked bookkeeping (`Bookkeeping<false>`) does, whatever order solve() applies its
operations in -- in particular the near-step flag, which only the packed form carries, must not leak into the recheck count
(a recheck after an accepted step below both the tolerance and kNearStep would otherwise end the frame at once).
Host build of the header through tests/emu/emu_bookkeeping.cpp (g++, no GPU)."""
import ctypes as C
import shutil
import subprocess
from pathlib import Path

import pytest

ROOT = Path(__file__).resolve().parent.parent
EMU = ROOT / "tests" / "emu"


@pytest.fixture(scope="module")
def lib(tmp_path_factory):
    if shutil.which("g++") is None:
        pytest.skip("needs g++")
    so = tmp_path_factory.mktemp("emu_bookkeeping") / "libdexr_emu_bookkeeping.so"
    cmd = ["g++", "-O0", "-std=c++17", "-fPIC", "-shared", f"-I{EMU / 'stub'}", "-o", str(so), str(EMU / "emu_bookkeeping.cpp")]
    res = subprocess.run(cmd, capture_output=True, text=True)
    assert res.returncode == 0, "g++ failed building the bookkeeping check:\n" + res.stderr[-4000:]
    lib = C.CDLL(str(so))
    lib.emu_bookkeeping_check.restype = C.c_int
    lib.emu_bookkeeping_first_recheck.restype = C.c_int
    return lib


def test_first_recheck_after_a_near_step_counts_one(lib):
    assert lib.emu_bookkeeping_first_recheck() == 1


@pytest.mark.parametrize("seed", range(8))
def test_packed_bookkeeping_matches_unpacked(lib, seed):
    err = C.create_string_buffer(300)
    rc = lib.emu_bookkeeping_check(C.c_uint(seed), C.c_int(4000), err, C.c_int(300))
    assert rc == 0, err.value.decode()
