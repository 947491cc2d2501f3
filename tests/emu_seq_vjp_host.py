"""Host emulation of backpropagation through the sequence solve (TEST INFRASTRUCTURE): builds tests/emu/emu_seq_vjp.cpp --
the fiber-warp emulation of tests/emu/emu_driver.cpp plus the recorded stream driver and the reverse-time VJP driver of
dex_retargeting_b200/csrc/dexr_kernels.cuh -- with g++ and calls its emu_solve_sequences_tape / emu_solve_sequences_vjp
through ctypes.  Used by tests/test_seq_vjp_emulation.py and, as the comparison, by tests/test_gpu_seq_vjp.py; never by the
product (the product path is the CUDA library only).  The build directory and the error type are those of
tests/emu_vjp_host.py."""
import ctypes as C
import subprocess
from functools import lru_cache

import numpy as np

from emu_eval_host import EMU, ROOT, EmulationError, _out_dir

SOURCES = [EMU / "emu_seq_vjp.cpp", EMU / "emu_driver.cpp", EMU / "warp_shim.h",
           ROOT / "dex_retargeting_b200" / "csrc" / "dexr_kernels.cuh", ROOT / "include" / "dexr.h"]


@lru_cache(maxsize=None)
def load(defines: tuple = ()):
    """defines: extra -D switches (the mutation checks of the test build variants of the kernel source with them)."""
    tag = "_".join(d.lower() for d in defines) or "default"
    so = _out_dir() / f"libdexr_emu_seq_vjp_{tag}.so"
    if not so.exists() or any(so.stat().st_mtime < p.stat().st_mtime for p in SOURCES):
        # -O0 as for emu_driver.cpp: the rendezvous protocol compares the call sites of the lanes
        cmd = ["g++", "-O0", "-std=c++17", "-fPIC", "-shared", f"-I{EMU / 'stub'}", *[f"-D{d}" for d in defines],
               "-o", str(so), str(EMU / "emu_seq_vjp.cpp")]
        res = subprocess.run(cmd, capture_output=True, text=True)
        if res.returncode != 0:
            raise RuntimeError("g++ failed building the host emulation:\n" + res.stderr[-4000:])
    lib = C.CDLL(str(so))
    lib.emu_solve_sequences_tape.restype = C.c_int
    lib.emu_solve_sequences_vjp.restype = C.c_int
    return lib


def _f32(a):
    return None if a is None else np.ascontiguousarray(a, dtype=np.float32)


def _ptr(a):
    return None if a is None else a.ctypes.data


def fresh_state(seq, S):
    """SeqRetargeting.make_stream_state as numpy arrays."""
    opt = seq.optimizer
    table = opt.build_table()
    return dict(last_qpos=np.tile(seq.joint_limits.mean(1).astype(np.float32), (S, 1)),
                filter_state=np.zeros((S, table.dof), np.float32), filter_init=np.zeros(S, np.uint8),
                projected=np.zeros((S, table.len_proj), np.uint8) if opt.retargeting_type == "DEXPILOT" else None,
                damping=np.zeros(S, np.float32))


def solve_sequences_tape(seq, keypoints, state=None, fixed_qpos=None, use_arrow=True, duo=False, defines=()):
    """Emulated dexr_solve_sequences_tape.  Returns (robot_qpos [S,T,dof], status [S,T], state, tape) with
    tape = dict(qpos [S,T,n], projected [S,T,len_proj] or None); `state` (numpy dict as for emu_host.solve_sequences) is
    updated in place."""
    from dex_retargeting_b200 import _native as N

    lib = load(tuple(defines))
    opt = seq.optimizer
    table, prm = opt.build_table(), opt.params(clip_init=True, lp_alpha=seq.low_pass_alpha)
    kp = _f32(keypoints)
    S, T = kp.shape[:2]
    state = fresh_state(seq, S) if state is None else state
    fixed = _f32(fixed_qpos) if table.n_fixed > 0 else None
    out = np.full((S, T, table.dof), np.nan, np.float32)
    status = np.zeros((S, T), np.int32)
    tape = dict(qpos=np.full((S, T, table.n_var), np.nan, np.float32),
                projected=np.full((S, T, table.len_proj), 7, np.uint8) if opt.retargeting_type == "DEXPILOT" else None)
    io = N.DexrSequences()
    io.keypoints, io.fixed_qpos, io.last_qpos = _ptr(kp), _ptr(fixed), _ptr(state["last_qpos"])
    io.filter_state, io.filter_init, io.projected = _ptr(state["filter_state"]), _ptr(state["filter_init"]), _ptr(state["projected"])
    io.robot_qpos_out, io.status_out, io.damping_state = _ptr(out), _ptr(status), _ptr(state.get("damping"))
    tp = N.DexrSequencesTape()
    tp.qpos, tp.projected = _ptr(tape["qpos"]), _ptr(tape["projected"])
    err = C.create_string_buffer(600)
    rc = lib.emu_solve_sequences_tape(C.byref(table), C.byref(prm), C.c_int(int(use_arrow)), C.byref(io), C.byref(tp),
                                      C.c_longlong(S), C.c_longlong(T), C.c_int(int(duo)), err, C.c_int(600))
    if rc != 0:
        raise EmulationError(rc, err.value.decode())
    return out, status, state, tape


def solve_sequences_vjp(seq, keypoints, tape_qpos, last_qpos0, filter_init0=None, tape_projected=None, grad_robot_qpos=None,
                        grad_last_qpos=None, grad_filter_state=None, fixed_qpos=None, spw=0, defines=(), null=(),
                        raw_hand=None):
    """Emulated dexr_solve_sequences_vjp.  Returns (grad_keypoints [S,T,21,3], grad_fixed [S,T,n_fixed] or None,
    grad_last_qpos0 [S,n], grad_filter_state0 [S,dof], status [S,T]); every output starts as NaN, so an entry the kernel does
    not write shows.  `spw` 1: one stream per warp (dexr_seq_vjp_kernel's other launch shape).  `null`: names of io fields
    passed as NULL (argument checks)."""
    from dex_retargeting_b200 import _native as N

    lib = load(tuple(defines))
    opt = seq.optimizer
    table, prm = opt.build_table(), opt.params(clip_init=True, lp_alpha=seq.low_pass_alpha, raw_hand=raw_hand)
    kp = _f32(keypoints)
    S, T = kp.shape[:2]
    arrays = dict(keypoints=kp, fixed_qpos=_f32(fixed_qpos) if table.n_fixed > 0 else None, last_qpos=_f32(last_qpos0),
                  filter_init=None if filter_init0 is None else np.ascontiguousarray(filter_init0, np.uint8),
                  qpos=_f32(tape_qpos), projected=None if tape_projected is None else np.ascontiguousarray(tape_projected, np.uint8),
                  grad_robot_qpos=_f32(grad_robot_qpos), grad_last_qpos_out=_f32(grad_last_qpos),
                  grad_filter_state_out=_f32(grad_filter_state))
    g_kp = np.full((S, T, N.NUM_KEYPOINTS, 3), np.nan, np.float32)
    g_fixed = np.full((S, T, table.n_fixed), np.nan, np.float32) if table.n_fixed else None
    g_last = np.full((S, table.n_var), np.nan, np.float32)
    g_filter = np.full((S, table.dof), np.nan, np.float32)
    status = np.full((S, T), -1, np.int32)
    io = N.DexrSequencesVjp()
    for k, a in arrays.items():
        setattr(io, k, None if k in null else _ptr(a))
    io.grad_keypoints, io.grad_fixed_qpos, io.grad_last_qpos = _ptr(g_kp), _ptr(g_fixed), _ptr(g_last)
    io.grad_filter_state, io.status_out = _ptr(g_filter), _ptr(status)
    err = C.create_string_buffer(600)
    rc = lib.emu_solve_sequences_vjp(C.byref(table), C.byref(prm), C.byref(io), C.c_longlong(S), C.c_longlong(T),
                                     C.c_int(int(spw)), err, C.c_int(600))
    if rc != 0:
        raise EmulationError(rc, err.value.decode())
    return g_kp, g_fixed, g_last, g_filter, status
