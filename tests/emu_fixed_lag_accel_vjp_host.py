"""Host emulation of the recording acceleration-penalised fixed-lag forward and of the backpropagation through it (TEST
INFRASTRUCTURE): builds tests/emu/emu_fixed_lag_accel_vjp.cpp -- the fiber-warp emulation of tests/emu/emu_driver.cpp plus
fixed_lag_tick<G, true, true>, the fixed_lag_vjp_* helpers with ACC and smooth_vjp_packed_stream<G, true, true> of
dex_retargeting_b200/csrc/dexr_kernels.cuh -- with g++ and calls it through ctypes.  Every buffer the driver may write lies
between guard words, checked after each call.  Used by tests/test_fixed_lag_accel_vjp_emulation.py and
tests/tools/emu_gpu_fixed_lag_accel_vjp.py; never by the product."""
import ctypes as C
import subprocess
from functools import lru_cache

import numpy as np

import emu_fixed_lag_accel_host as FA
import emu_fixed_lag_vjp_host as FV
from emu_eval_host import EMU, ROOT, EmulationError, _out_dir
from emu_packed_host import Guarded

SOURCES = [EMU / "emu_fixed_lag_accel_vjp.cpp", EMU / "emu_driver.cpp", EMU / "warp_shim.h",
           ROOT / "dex_retargeting_b200" / "csrc" / "dexr_kernels.cuh", ROOT / "include" / "dexr.h"]
GRADS_IN = FV.GRADS_IN + ("grad_prev_qpos_out",)
STATE = FA.STATE


@lru_cache(maxsize=None)
def load():
    so = _out_dir() / "libdexr_emu_fixed_lag_accel_vjp.so"
    if not so.exists() or any(so.stat().st_mtime < p.stat().st_mtime for p in SOURCES):
        # -O0 as for emu_driver.cpp: the rendezvous protocol compares the call sites of the lanes
        cmd = ["g++", "-O0", "-std=c++17", "-fPIC", "-shared", f"-I{EMU / 'stub'}", "-o", str(so),
               str(EMU / "emu_fixed_lag_accel_vjp.cpp")]
        res = subprocess.run(cmd, capture_output=True, text=True)
        if res.returncode != 0:
            raise RuntimeError("g++ failed building the host emulation:\n" + res.stderr[-4000:])
    lib = C.CDLL(str(so))
    lib.emu_fixed_lag_step_accel_tape.restype = C.c_int
    lib.emu_fixed_lag_step_accel_vjp.restype = C.c_int
    lib.emu_fixed_lag_accel_vjp_workspace_bytes.restype = C.c_size_t
    lib.emu_fixed_lag_accel_vjp_sizeof.restype = C.c_size_t
    lib.emu_fixed_lag_vjp_sizeof.restype = C.c_size_t
    return lib


def workspace_bytes_of(table, S, lag):
    return int(load().emu_fixed_lag_accel_vjp_workspace_bytes(C.byref(table), C.c_longlong(S), C.c_int(lag)))


def workspace_bytes(seq, S, lag):
    return workspace_bytes_of(seq.optimizer.build_table(), S, lag)


def _f32(a):
    return None if a is None else np.ascontiguousarray(a, np.float32)


def fixed_lag_step_accel_tape(seq, keypoints, state, fixed_qpos=None, smooth_weight=-1.0, flush=False):
    """Emulated dexr_fixed_lag_step_accel_tape: keypoints [S,K,21,3] (None: K = 0), `state` an accelerated numpy state
    (emu_fixed_lag_accel_host.fresh_state) updated in place.  Returns emu_fixed_lag_accel_host.fixed_lag_step's outputs plus
    tape_qpos [S,K,L+1,n] and tape_projected [S,K,len_proj] (or None)."""
    from dex_retargeting_b200 import _native as N

    lib = load()
    opt = seq.optimizer
    table = opt.build_table()
    prm = opt.params(clip_init=True, lp_alpha=seq.low_pass_alpha)
    S, L = state["last_qpos"].shape[0], state["lag"]
    K = 0 if keypoints is None else keypoints.shape[1]
    kp, fx = _f32(keypoints), (_f32(fixed_qpos) if table.n_fixed else None)
    guards = {k: Guarded(state[k], np.array(-9 if state[k].dtype == np.int32 else
                                            (0xAB if state[k].dtype == np.uint8 else -7.0), state[k].dtype))
              for k in STATE if state.get(k) is not None}
    outs = dict(qpos=Guarded(np.full((S, K, table.n_var), np.nan, np.float32), np.float32(-7.0)),
                robot_qpos=Guarded(np.full((S, K, table.dof), np.nan, np.float32), np.float32(-7.0)),
                status=Guarded(np.full((S, K), -1, np.int32), np.int32(-9)),
                tape_qpos=Guarded(np.full((S, K, L + 1, table.n_var), np.nan, np.float32), np.float32(-7.0)))
    if table.len_proj:
        outs["tape_projected"] = Guarded(np.full((S, K, table.len_proj), 0xAB, np.uint8), np.uint8(0xCD))
    if flush:
        outs.update(flush_qpos=Guarded(np.full((S, L, table.n_var), -3.0, np.float32), np.float32(-7.0)),
                    flush_robot_qpos=Guarded(np.full((S, L, table.dof), -3.0, np.float32), np.float32(-7.0)),
                    flush_count=Guarded(np.full(S, -1, np.int32), np.int32(-9)))
    nbytes = FA.workspace_bytes(seq, S, L)
    ws = Guarded(np.full(max(nbytes // 4, 1), np.nan, np.float32), np.float32(-7.0))
    io = N.DexrFixedLag()
    io.keypoints = None if kp is None else kp.ctypes.data
    io.fixed_qpos = None if fx is None else fx.ctypes.data
    for k, g in guards.items():
        if k not in ("prev_qpos", "has_prev"):
            setattr(io, k, g.ptr())
    for k, f in (("qpos", "qpos_out"), ("robot_qpos", "robot_qpos_out"), ("status", "status_out"),
                 ("flush_qpos", "flush_qpos_out"), ("flush_robot_qpos", "flush_robot_qpos_out"),
                 ("flush_count", "flush_count_out")):
        if k in outs:
            setattr(io, f, outs[k].ptr())
    io.lag, io.smooth_weight = L, smooth_weight
    io.workspace, io.workspace_bytes = ws.ptr(), nbytes
    acc = FA._accel_struct(state["accel_weight"], guards["prev_qpos"].ptr(), guards["has_prev"].ptr())
    tp = N.DexrFixedLagTape()
    tp.qpos = outs["tape_qpos"].ptr()
    tp.projected = outs["tape_projected"].ptr() if "tape_projected" in outs else None
    err = C.create_string_buffer(600)
    rc = lib.emu_fixed_lag_step_accel_tape(C.byref(table), C.byref(prm), C.byref(io), C.byref(acc), C.byref(tp),
                                           C.c_longlong(S), C.c_longlong(K), err, C.c_int(600))
    if rc != 0:
        raise EmulationError(rc, err.value.decode())
    for name, b in list(outs.items()) + list(guards.items()) + [("workspace", ws)]:
        b.check(name)
    for k, g in guards.items():
        state[k][...] = g.a
    r = {k: g.a for k, g in outs.items()}
    r.setdefault("tape_projected", None)
    return r


def fixed_lag_accel_vjp(seq, keypoints, state0, tape_qpos, tape_projected=None, fixed_qpos=None, flushed=False,
                        smooth_weight=-1.0, null=(), workspace_bytes=None, num_ticks=None, accel_weight=None, **grads):
    """Emulated dexr_fixed_lag_step_accel_vjp: emu_fixed_lag_vjp_host.fixed_lag_vjp's arguments with `state0` the accelerated
    numpy state before the forward (its accel_weight, prev_qpos and has_prev; `accel_weight` overrides c) and
    grad_prev_qpos_out among the cotangents.  Returns fixed_lag_vjp's dict plus grad_prev_qpos."""
    from dex_retargeting_b200 import _native as N

    lib = load()
    opt = seq.optimizer
    table = opt.build_table()
    prm = opt.params(clip_init=True, lp_alpha=seq.low_pass_alpha)
    S, L = state0["last_qpos"].shape[0], state0["lag"]
    K = 0 if keypoints is None else keypoints.shape[1]
    n, nf = table.n_var, table.n_fixed
    inputs = dict(keypoints=_f32(keypoints), fixed_qpos=_f32(fixed_qpos) if nf else None)
    for k in STATE:
        v = state0.get(k)
        inputs[k] = None if v is None else np.ascontiguousarray(v)
    for k in GRADS_IN:
        inputs[k] = _f32(grads.get(k))
    tq = _f32(tape_qpos)
    tpj = None if tape_projected is None else np.ascontiguousarray(tape_projected, np.uint8)
    before = {k: None if v is None else v.copy() for k, v in inputs.items()}
    nan = np.float32(np.nan)
    outs = dict(grad_keypoints=Guarded(np.full((S, K, 21, 3), nan, np.float32), np.float32(-7.0)),
                grad_fixed_qpos=Guarded(np.full((S, K, nf), nan, np.float32), np.float32(-7.0)),
                grad_last_qpos=Guarded(np.full((S, n), nan, np.float32), np.float32(-7.0)),
                grad_window_keypoints=Guarded(np.full((S, L + 1, 21, 3), nan, np.float32), np.float32(-7.0)),
                grad_window_fixed_qpos=Guarded(np.full((S, L + 1, nf), nan, np.float32), np.float32(-7.0)),
                grad_window_qpos=Guarded(np.full((S, L + 1, n), nan, np.float32), np.float32(-7.0)),
                status_out=Guarded(np.full((S, K), -1, np.int32), np.int32(-9)),
                grad_prev_qpos=Guarded(np.full((S, n), nan, np.float32), np.float32(-7.0)))
    nbytes = workspace_bytes_of(table, S, L) if workspace_bytes is None else workspace_bytes
    ws = Guarded(np.full(max(nbytes // 4, 1), nan, np.float32), np.float32(-7.0))
    io = N.DexrFixedLagVjp()
    acc = N.DexrFixedLagAccelVjp()
    acc_fields = ("prev_qpos", "has_prev", "grad_prev_qpos_out")
    for k, v in inputs.items():
        setattr(acc if k in acc_fields else io, k, None if v is None or k in null else v.ctypes.data)
    io.tape.qpos = None if tq is None or "tape.qpos" in null else tq.ctypes.data
    io.tape.projected = None if tpj is None or "tape.projected" in null else tpj.ctypes.data
    for k, g in outs.items():
        setattr(acc if k == "grad_prev_qpos" else io, k, None if k in null or (nf == 0 and "fixed" in k) else g.ptr())
    acc.accel_weight = state0["accel_weight"] if accel_weight is None else accel_weight
    io.lag = L
    io.flushed = int(bool(flushed))
    io.smooth_weight = smooth_weight
    io.workspace = None if "workspace" in null else ws.ptr()
    io.workspace_bytes = nbytes
    err = C.create_string_buffer(600)
    rc = lib.emu_fixed_lag_step_accel_vjp(C.byref(table), C.byref(prm), C.byref(io), C.byref(acc), C.c_longlong(S),
                                          C.c_longlong(K if num_ticks is None else num_ticks), err, C.c_int(600))
    if rc != 0:
        raise EmulationError(rc, err.value.decode())
    for name, b in list(outs.items()) + [("workspace", ws)]:
        b.check(name)
    for k, v in inputs.items():
        if v is not None:
            np.testing.assert_array_equal(v, before[k], err_msg=f"{k} was written")
    r = {k: g.a for k, g in outs.items()}
    r["status"] = r.pop("status_out")
    return r
