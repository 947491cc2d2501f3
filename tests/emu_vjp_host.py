"""Host emulation of backpropagation through the solve (TEST INFRASTRUCTURE): builds tests/emu/emu_vjp.cpp -- the fiber-warp
emulation of tests/emu/emu_driver.cpp plus the VJP driver of dex_retargeting_b200/csrc/dexr_kernels.cuh -- with g++ and calls
its emu_solve_vjp through ctypes.  Used by tests/test_vjp_emulation.py and, as the comparison, by tests/test_gpu_vjp.py; never
by the product (the product path is the CUDA library only).  The build directory and the error type are those of
tests/emu_eval_host.py."""
import ctypes as C
import subprocess
from functools import lru_cache

import numpy as np

from emu_eval_host import EMU, ROOT, EmulationError, _out_dir

SOURCES = [EMU / "emu_vjp.cpp", EMU / "emu_driver.cpp", EMU / "warp_shim.h",
           ROOT / "dex_retargeting_b200" / "csrc" / "dexr_kernels.cuh", ROOT / "include" / "dexr.h"]


@lru_cache(maxsize=None)
def load():
    so = _out_dir() / "libdexr_emu_vjp.so"
    if not so.exists() or any(so.stat().st_mtime < p.stat().st_mtime for p in SOURCES):
        # -O0 as for emu_driver.cpp: the rendezvous protocol compares the call sites of the lanes
        cmd = ["g++", "-O0", "-std=c++17", "-fPIC", "-shared", f"-I{EMU / 'stub'}", "-o", str(so), str(EMU / "emu_vjp.cpp")]
        res = subprocess.run(cmd, capture_output=True, text=True)
        if res.returncode != 0:
            raise RuntimeError("g++ failed building the host emulation:\n" + res.stderr[-4000:])
    lib = C.CDLL(str(so))
    lib.emu_solve_vjp.restype = C.c_int
    return lib


def solve_vjp(opt, grad_qpos, qpos, keypoints=None, ref_value=None, fixed_qpos=None, last_qpos=None, projected=None,
              want=("targets", "fixed", "last"), raw_hand=None, null_grad_qpos=False):
    """Emulated dexr_solve_vjp for an Optimizer of the host mirror (table and parameters as for emu_eval_host.eval_objective).
    Returns (grad_targets [B,21,3] or [B,m,3], grad_fixed [B,n_fixed] or None, grad_last [B,n] or None, status [B]); every
    requested output starts as NaN, so an entry the kernel does not write shows.  `projected` is read only."""
    from dex_retargeting_b200 import _native as N

    lib = load()
    table, prm = opt.build_table(), opt.params(raw_hand=raw_hand)

    def f32(a):
        return None if a is None else np.ascontiguousarray(a, dtype=np.float32)

    def ptr(a):
        return None if a is None else a.ctypes.data

    x, gq = f32(qpos), f32(grad_qpos)
    B = 0 if x is None else x.shape[0]
    kp, ref, fixed, last = f32(keypoints), f32(ref_value), f32(fixed_qpos), f32(last_qpos)
    g_tgt = None
    if "targets" in want:
        g_tgt = np.full((B, N.NUM_KEYPOINTS, 3) if kp is not None else (B, table.n_res, 3), np.nan, np.float32)
    g_fixed = np.full((B, table.n_fixed), np.nan, np.float32) if "fixed" in want and table.n_fixed else None
    g_last = np.full((B, table.n_var), np.nan, np.float32) if "last" in want and last is not None else None
    status = np.full(B, -1, np.int32)
    io = N.DexrVjp()
    io.keypoints, io.ref_value, io.fixed_qpos, io.qpos, io.last_qpos = ptr(kp), ptr(ref), ptr(fixed), ptr(x), ptr(last)
    io.projected, io.grad_qpos = ptr(projected), None if null_grad_qpos else ptr(gq)
    io.grad_keypoints = ptr(g_tgt) if kp is not None else None
    io.grad_ref_value = ptr(g_tgt) if kp is None else None
    io.grad_fixed_qpos, io.grad_last_qpos, io.status_out = ptr(g_fixed), ptr(g_last), ptr(status)
    err = C.create_string_buffer(600)
    rc = lib.emu_solve_vjp(C.byref(table), C.byref(prm), C.byref(io), C.c_longlong(B), err, C.c_int(600))
    if rc != 0:
        raise EmulationError(rc, err.value.decode())
    return g_tgt, g_fixed, g_last, status
