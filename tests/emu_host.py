"""Host emulation of the CUDA solver source (TEST INFRASTRUCTURE): builds tests/emu/emu_driver.cpp -- which compiles
dex_retargeting_b200/csrc/dexr_kernels.cuh itself through tests/emu/warp_shim.h -- with g++ and calls it through ctypes.
Used by tests/test_solver_host_emulation.py; never by the product (the product path is the CUDA library only)."""
import ctypes as C
import subprocess
from functools import lru_cache
from pathlib import Path

import numpy as np

ROOT = Path(__file__).resolve().parent.parent
EMU = ROOT / "tests" / "emu"
OUT = EMU / "_build"
SOURCES = [EMU / "emu_driver.cpp", EMU / "warp_shim.h", ROOT / "dex_retargeting_b200" / "csrc" / "dexr_kernels.cuh",
           ROOT / "include" / "dexr.h"]


@lru_cache(maxsize=None)
def load(defines: tuple = ()):
    """defines: compile-time experiment switches, e.g. ("DEXR_EXP_FASTSINCOS",)."""
    OUT.mkdir(exist_ok=True)
    tag = "_".join(d.replace("DEXR_EXP_", "").lower() for d in defines) or "default"
    so = OUT / f"libdexr_emu_{tag}.so"
    if not so.exists() or any(so.stat().st_mtime < p.stat().st_mtime for p in SOURCES):
        # -O0: the rendezvous protocol compares the call sites of the lanes, and optimising host compilers duplicate calls
        # (jump threading) -- they do not know that a warp collective is convergent
        cmd = ["g++", "-O0", "-std=c++17", "-fPIC", "-shared", f"-I{EMU / 'stub'}", *[f"-D{d}" for d in defines],
               "-o", str(so), str(EMU / "emu_driver.cpp")]
        res = subprocess.run(cmd, capture_output=True, text=True)
        if res.returncode != 0:
            raise RuntimeError("g++ failed building the host emulation:\n" + res.stderr[-4000:])
    lib = C.CDLL(str(so))
    lib.emu_solve_frames.restype = C.c_int
    lib.emu_rounds.restype = C.c_longlong
    return lib


def solve_frames(opt, last_qpos, keypoints=None, ref_value=None, fixed_qpos=None, projected=None, defines=(), use_arrow=True,
                 clip_init=False, want_robot_qpos=False, raw_hand=None, damping=None):
    """Emulated dexr_solve_frames for an Optimizer of the host mirror.  Returns (qpos [B,n], status [B], cost [B])
    (+ the full joint vector [B,dof] with want_robot_qpos).  `damping`: float32 [B] in/out (dexr_frames_t.damping_io)."""
    from dex_retargeting_b200 import _native as N

    lib = load(tuple(defines))
    table, prm = opt.build_table(), opt.params(clip_init=clip_init, raw_hand=raw_hand)
    B, n = last_qpos.shape[0], table.n_var

    def f32(a):
        return None if a is None else np.ascontiguousarray(a, dtype=np.float32)

    kp, ref, last, fixed = f32(keypoints), f32(ref_value), f32(last_qpos), f32(fixed_qpos)
    assert (kp is None) != (ref is None)
    out = np.full((B, n), np.nan, np.float32)
    status = np.zeros(B, np.int32)
    cost = np.zeros(B, np.float32)
    err = C.create_string_buffer(600)

    def ptr(a):
        return None if a is None else a.ctypes.data

    full = np.zeros((B, table.dof), np.float32) if want_robot_qpos else None
    io = N.DexrFrames()
    io.keypoints, io.ref_value, io.last_qpos, io.fixed_qpos = ptr(kp), ptr(ref), ptr(last), ptr(fixed)
    io.projected, io.qpos_out, io.robot_qpos_out = ptr(projected), ptr(out), ptr(full)
    io.status_out, io.cost_out, io.damping_io = ptr(status), ptr(cost), ptr(damping)
    rc = lib.emu_solve_frames(C.byref(table), C.byref(prm), C.c_int(int(use_arrow)), C.byref(io), C.c_longlong(B), err,
                              C.c_int(600))
    if rc != 0:
        raise RuntimeError(f"host emulation failed ({rc}): {err.value.decode()}")
    return (out, status, cost, full) if want_robot_qpos else (out, status, cost)


def solve_sequences(seq, keypoints, state=None, defines=(), use_arrow=True, raw_hand=None, duo=False, fixed_qpos=None):
    """Emulated dexr_solve_sequences for a SeqRetargeting of the host mirror: keypoints [S,T,21,3] (+ fixed_qpos [S,T,n_fixed]
    when the robot has fixed joints) -> filtered robot qpos [S,T,dof]; `state` = dict(last_qpos, filter_state, filter_init,
    projected, damping) carried between calls (created if None).
    `duo`: the scarce-streams mode of the 16-lane solver (both half-warps on one stream, residual passes split)."""
    from dex_retargeting_b200 import _native as N

    lib = load(tuple(defines))
    opt = seq.optimizer
    table, prm = opt.build_table(), opt.params(clip_init=True, lp_alpha=seq.low_pass_alpha, raw_hand=raw_hand)
    kp = np.ascontiguousarray(keypoints, dtype=np.float32)
    S, T = kp.shape[:2]
    fixed = None
    if table.n_fixed > 0:
        assert fixed_qpos is not None, f"robot has {table.n_fixed} fixed joints but no fixed_qpos is given"
        fixed = np.ascontiguousarray(fixed_qpos, dtype=np.float32)
        assert fixed.shape == (S, T, table.n_fixed), fixed.shape
    if state is None:  # SeqRetargeting.make_stream_state: mid-range warm start, filter not initialised, no projection
        state = dict(last_qpos=np.tile(seq.joint_limits.mean(1).astype(np.float32), (S, 1)),
                     filter_state=np.zeros((S, table.dof), np.float32), filter_init=np.zeros(S, np.uint8),
                     projected=np.zeros((S, table.len_proj), np.uint8) if opt.retargeting_type == "DEXPILOT" else None,
                     damping=np.zeros(S, np.float32))
    out = np.full((S, T, table.dof), np.nan, np.float32)
    status = np.zeros((S, T), np.int32)
    io = N.DexrSequences()
    io.keypoints, io.last_qpos = kp.ctypes.data, state["last_qpos"].ctypes.data
    if fixed is not None:
        io.fixed_qpos = fixed.ctypes.data
    io.filter_state, io.filter_init = state["filter_state"].ctypes.data, state["filter_init"].ctypes.data
    io.projected = state["projected"].ctypes.data if state["projected"] is not None else None
    io.robot_qpos_out, io.status_out = out.ctypes.data, status.ctypes.data
    if state.get("damping") is not None:
        io.damping_state = state["damping"].ctypes.data
    err = C.create_string_buffer(600)
    lib.emu_solve_sequences.restype = C.c_int
    rc = lib.emu_solve_sequences(C.byref(table), C.byref(prm), C.c_int(int(use_arrow)), C.byref(io), C.c_longlong(S),
                                 C.c_longlong(T), C.c_int(int(duo)), err, C.c_int(600))
    if rc != 0:
        raise RuntimeError(f"host emulation failed ({rc}): {err.value.decode()}")
    return out, status, state
