"""Host emulation of the per-frame Jacobians of the solve (TEST INFRASTRUCTURE): builds tests/emu/emu_jacobian.cpp -- the
fiber-warp emulation of tests/emu/emu_driver.cpp plus the Jacobian driver of dex_retargeting_b200/csrc/dexr_kernels.cuh --
with g++ and calls its emu_solve_jacobian through ctypes.  Used by tests/test_jacobian_emulation.py and, as the comparison,
by tests/test_gpu_jacobian.py; never by the product (the product path is the CUDA library only).  The build directory and
the error type are those of tests/emu_eval_host.py."""
import ctypes as C
import subprocess
from functools import lru_cache

import numpy as np

from emu_eval_host import EMU, ROOT, EmulationError, _out_dir

SOURCES = [EMU / "emu_jacobian.cpp", EMU / "emu_driver.cpp", EMU / "warp_shim.h",
           ROOT / "dex_retargeting_b200" / "csrc" / "dexr_kernels.cuh", ROOT / "include" / "dexr.h"]


@lru_cache(maxsize=None)
def load():
    so = _out_dir() / "libdexr_emu_jacobian.so"
    if not so.exists() or any(so.stat().st_mtime < p.stat().st_mtime for p in SOURCES):
        # -O0 as for emu_driver.cpp: the rendezvous protocol compares the call sites of the lanes
        cmd = ["g++", "-O0", "-std=c++17", "-fPIC", "-shared", f"-I{EMU / 'stub'}", "-o", str(so),
               str(EMU / "emu_jacobian.cpp")]
        res = subprocess.run(cmd, capture_output=True, text=True)
        if res.returncode != 0:
            raise RuntimeError("g++ failed building the host emulation:\n" + res.stderr[-4000:])
    lib = C.CDLL(str(so))
    lib.emu_solve_jacobian.restype = C.c_int
    return lib


def solve_jacobian(opt, qpos, keypoints=None, ref_value=None, fixed_qpos=None, last_qpos=None, projected=None,
                   want=("targets", "fixed", "last"), raw_hand=None):
    """Emulated dexr_solve_jacobian for an Optimizer of the host mirror (table and parameters as for
    emu_eval_host.eval_objective).  Returns (jac_targets [B,n,21,3] or [B,n,m,3], jac_fixed [B,n,n_fixed] or None,
    jac_last [B,n,n] or None, status [B]); every requested output starts as NaN, so an entry the kernel does not write
    shows.  `projected` is read only."""
    from dex_retargeting_b200 import _native as N

    lib = load()
    table, prm = opt.build_table(), opt.params(raw_hand=raw_hand)

    def f32(a):
        return None if a is None else np.ascontiguousarray(a, dtype=np.float32)

    def ptr(a):
        return None if a is None else a.ctypes.data

    x = f32(qpos)
    B = 0 if x is None else x.shape[0]
    n = table.n_var
    kp, ref, fixed, last = f32(keypoints), f32(ref_value), f32(fixed_qpos), f32(last_qpos)
    j_tgt = None
    if "targets" in want:
        j_tgt = np.full((B, n, N.NUM_KEYPOINTS, 3) if kp is not None else (B, n, table.n_res, 3), np.nan, np.float32)
    j_fixed = np.full((B, n, table.n_fixed), np.nan, np.float32) if "fixed" in want and table.n_fixed else None
    j_last = np.full((B, n, n), np.nan, np.float32) if "last" in want and last is not None else None
    status = np.full(B, -1, np.int32)
    io = N.DexrJacobian()
    io.keypoints, io.ref_value, io.fixed_qpos, io.qpos, io.last_qpos = ptr(kp), ptr(ref), ptr(fixed), ptr(x), ptr(last)
    io.projected = ptr(projected)
    io.jac_keypoints = ptr(j_tgt) if kp is not None else None
    io.jac_ref_value = ptr(j_tgt) if kp is None else None
    io.jac_fixed_qpos, io.jac_last_qpos, io.status_out = ptr(j_fixed), ptr(j_last), ptr(status)
    err = C.create_string_buffer(600)
    rc = lib.emu_solve_jacobian(C.byref(table), C.byref(prm), C.byref(io), C.c_longlong(B), err, C.c_int(600))
    if rc != 0:
        raise EmulationError(rc, err.value.decode())
    return j_tgt, j_fixed, j_last, status
