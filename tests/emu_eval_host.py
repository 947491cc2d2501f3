"""Host emulation of the objective evaluation (TEST INFRASTRUCTURE): builds tests/emu/emu_eval.cpp -- the fiber-warp emulation
of tests/emu/emu_driver.cpp plus the evaluation driver of dex_retargeting_b200/csrc/dexr_kernels.cuh -- with g++ and calls its
emu_eval_objective through ctypes.  Used by tests/test_objective_emulation.py and, as the comparison, by
tests/test_gpu_objective.py; never by the product (the product path is the CUDA library only)."""
import ctypes as C
import os
import subprocess
import tempfile
from functools import lru_cache
from pathlib import Path

import numpy as np

ROOT = Path(__file__).resolve().parent.parent
EMU = ROOT / "tests" / "emu"
SOURCES = [EMU / "emu_eval.cpp", EMU / "emu_driver.cpp", EMU / "warp_shim.h",
           ROOT / "dex_retargeting_b200" / "csrc" / "dexr_kernels.cuh", ROOT / "include" / "dexr.h"]


def _out_dir() -> Path:
    """tests/emu/_build, or a directory under the temporary directory when the tree is read-only."""
    out = EMU / "_build"
    try:
        out.mkdir(exist_ok=True)
        if os.access(out, os.W_OK):
            return out
    except OSError:
        pass
    out = Path(tempfile.gettempdir()) / f"dexr_emu_build_{os.getuid()}"
    out.mkdir(exist_ok=True)
    return out


@lru_cache(maxsize=None)
def load(defines: tuple = ()):
    """defines: compile-time experiment switches, e.g. ("DEXR_EXP_FASTSINCOS",)."""
    tag = "_".join(d.replace("DEXR_EXP_", "").lower() for d in defines) or "default"
    so = _out_dir() / f"libdexr_emu_eval_{tag}.so"
    if not so.exists() or any(so.stat().st_mtime < p.stat().st_mtime for p in SOURCES):
        # -O0 as for emu_driver.cpp: the rendezvous protocol compares the call sites of the lanes
        cmd = ["g++", "-O0", "-std=c++17", "-fPIC", "-shared", f"-I{EMU / 'stub'}", *[f"-D{d}" for d in defines],
               "-o", str(so), str(EMU / "emu_eval.cpp")]
        res = subprocess.run(cmd, capture_output=True, text=True)
        if res.returncode != 0:
            raise RuntimeError("g++ failed building the host emulation:\n" + res.stderr[-4000:])
    lib = C.CDLL(str(so))
    lib.emu_eval_objective.restype = C.c_int
    return lib


class EmulationError(RuntimeError):
    """The emulated entry point rejected its arguments or failed: `code` is its return value (-1 = DEXR_E_INVALID)."""

    def __init__(self, code, msg):
        super().__init__(f"host emulation failed ({code}): {msg}")
        self.code, self.msg = code, msg


def eval_objective(opt, qpos, keypoints=None, ref_value=None, fixed_qpos=None, last_qpos=None, projected=None, raw_hand=None,
                   want_grad=True, defines=()):
    """Emulated dexr_eval_objective for an Optimizer of the host mirror.  Returns (loss [B], cost [B], grad [B,n] or None);
    `projected` (uint8 [B,len_proj]) is read and updated in place."""
    from dex_retargeting_b200 import _native as N

    lib = load(tuple(defines))
    table, prm = opt.build_table(), opt.params(raw_hand=raw_hand)

    def f32(a):
        return None if a is None else np.ascontiguousarray(a, dtype=np.float32)

    def ptr(a):
        return None if a is None else a.ctypes.data

    x = f32(qpos)
    B = 0 if x is None else x.shape[0]
    kp, ref, fixed, last = f32(keypoints), f32(ref_value), f32(fixed_qpos), f32(last_qpos)
    loss, cost = np.full(B, np.nan, np.float32), np.full(B, np.nan, np.float32)
    grad = np.full((B, table.n_var), np.nan, np.float32) if want_grad else None
    io = N.DexrEval()
    io.keypoints, io.ref_value, io.fixed_qpos, io.qpos, io.last_qpos = ptr(kp), ptr(ref), ptr(fixed), ptr(x), ptr(last)
    io.projected, io.loss_out, io.cost_out, io.grad_out = ptr(projected), ptr(loss), ptr(cost), ptr(grad)
    err = C.create_string_buffer(600)
    rc = lib.emu_eval_objective(C.byref(table), C.byref(prm), C.byref(io), C.c_longlong(B), err, C.c_int(600))
    if rc != 0:
        raise EmulationError(rc, err.value.decode())
    return loss, cost, grad
