"""Host emulation of acceleration-penalised fixed-lag smoothing (TEST INFRASTRUCTURE): builds
tests/emu/emu_fixed_lag_accel.cpp -- the fiber-warp emulation of tests/emu/emu_driver.cpp plus fixed_lag_tick /
fixed_lag_flush / smooth_packed_stream of dex_retargeting_b200/csrc/dexr_kernels.cuh with the pre-anchor -- with g++ and calls
emu_fixed_lag_step_accel and emu_smooth_packed_pre_anchor through ctypes.  Every buffer the driver may write, the stream
state included, lies between guard words, checked after each call.  Used by tests/test_fixed_lag_accel_emulation.py and
tests/tools/emu_gpu_fixed_lag_accel.py; never by the product."""
import ctypes as C
import subprocess
from functools import lru_cache

import numpy as np

import emu_fixed_lag_host as FL
import emu_smooth_accel_host as SA
from emu_eval_host import EMU, ROOT, EmulationError, _out_dir
from emu_packed_host import Guarded

SOURCES = [EMU / "emu_fixed_lag_accel.cpp", EMU / "emu_driver.cpp", EMU / "warp_shim.h",
           ROOT / "dex_retargeting_b200" / "csrc" / "dexr_kernels.cuh", ROOT / "include" / "dexr.h"]
STATE = FL.STATE + ("prev_qpos", "has_prev")


@lru_cache(maxsize=None)
def load():
    so = _out_dir() / "libdexr_emu_fixed_lag_accel.so"
    if not so.exists() or any(so.stat().st_mtime < p.stat().st_mtime for p in SOURCES):
        # -O0 as for emu_driver.cpp: the rendezvous protocol compares the call sites of the lanes
        cmd = ["g++", "-O0", "-std=c++17", "-fPIC", "-shared", f"-I{EMU / 'stub'}", "-o", str(so),
               str(EMU / "emu_fixed_lag_accel.cpp")]
        res = subprocess.run(cmd, capture_output=True, text=True)
        if res.returncode != 0:
            raise RuntimeError("g++ failed building the host emulation:\n" + res.stderr[-4000:])
    lib = C.CDLL(str(so))
    lib.emu_fixed_lag_step_accel.restype = C.c_int
    lib.emu_smooth_packed_pre_anchor.restype = C.c_int
    lib.emu_fixed_lag_accel_workspace_bytes.restype = C.c_size_t
    return lib


def workspace_bytes(seq, S, lag):
    return int(load().emu_fixed_lag_accel_workspace_bytes(C.byref(seq.optimizer.build_table()), C.c_longlong(S),
                                                          C.c_int(lag)))


def fresh_state(seq, S, lag, accel_weight):
    """SeqRetargeting.make_fixed_lag_state(S, lag, accel_weight) as numpy arrays (plus "lag" and "accel_weight")."""
    st = FL.fresh_state(seq, S, lag)
    st.update(accel_weight=float(accel_weight), prev_qpos=np.zeros((S, seq.optimizer.opt_dof), np.float32),
              has_prev=np.zeros(S, np.int32))
    return st


def _accel_struct(c, prev, has):
    from dex_retargeting_b200 import _native as N

    acc = N.DexrFixedLagAccel()
    acc.accel_weight = c
    acc.prev_qpos = prev
    acc.has_prev = has
    return acc


def fixed_lag_step(seq, keypoints, state, fixed_qpos=None, smooth_weight=-1.0, flush=False, null=(), workspace_bytes=None,
                   params=None, num_streams=None, num_ticks=None, lag=None, accel_weight=None):
    """Emulated dexr_fixed_lag_step_accel (arguments and result as emu_fixed_lag_host.fixed_lag_step; the state also holds
    accel_weight, prev_qpos and has_prev, updated in place; `accel_weight` overrides the state's for the call)."""
    from dex_retargeting_b200 import _native as N

    lib = load()
    opt = seq.optimizer
    table = opt.build_table()
    prm = opt.params(clip_init=True, lp_alpha=seq.low_pass_alpha) if params is None else params
    S = state["last_qpos"].shape[0]
    L = state["lag"]
    K = 0 if keypoints is None else keypoints.shape[1]
    kp = None if keypoints is None else np.ascontiguousarray(keypoints, np.float32)
    fx = None if fixed_qpos is None or not table.n_fixed else np.ascontiguousarray(fixed_qpos, np.float32)
    inputs = dict(keypoints=kp, fixed_qpos=fx)
    before = {k: None if v is None else v.copy() for k, v in inputs.items()}
    guards = {}
    for k in STATE:  # the state is written in place: guarded too
        v = state.get(k)
        if v is not None:
            guards[k] = Guarded(v, np.array(-9 if v.dtype == np.int32 else (0xAB if v.dtype == np.uint8 else -7.0), v.dtype))
    outs = dict(qpos=Guarded(np.full((S, K, table.n_var), np.nan, np.float32), np.float32(-7.0)),
                robot_qpos=Guarded(np.full((S, K, table.dof), np.nan, np.float32), np.float32(-7.0)),
                status=Guarded(np.full((S, K), -1, np.int32), np.int32(-9)))
    if flush:
        outs.update(flush_qpos=Guarded(np.full((S, L, table.n_var), -3.0, np.float32), np.float32(-7.0)),
                    flush_robot_qpos=Guarded(np.full((S, L, table.dof), -3.0, np.float32), np.float32(-7.0)),
                    flush_count=Guarded(np.full(S, -1, np.int32), np.int32(-9)))
    nbytes = int(lib.emu_fixed_lag_accel_workspace_bytes(C.byref(table), C.c_longlong(S), C.c_int(L))) \
        if workspace_bytes is None else workspace_bytes
    ws = Guarded(np.full(max(nbytes // 4, 1), np.nan, np.float32), np.float32(-7.0))
    io = N.DexrFixedLag()
    for k, v in inputs.items():
        setattr(io, k, None if v is None or k in null else v.ctypes.data)
    for k, g in guards.items():
        if k in FL.STATE:
            setattr(io, k, None if k in null else g.ptr())
    for k, f in (("qpos", "qpos_out"), ("robot_qpos", "robot_qpos_out"), ("status", "status_out"),
                 ("flush_qpos", "flush_qpos_out"), ("flush_robot_qpos", "flush_robot_qpos_out"),
                 ("flush_count", "flush_count_out")):
        if k in outs:
            setattr(io, f, None if f in null else outs[k].ptr())
    io.lag = L if lag is None else lag
    io.smooth_weight = smooth_weight
    io.workspace = None if "workspace" in null else ws.ptr()
    io.workspace_bytes = nbytes
    acc = _accel_struct(state["accel_weight"] if accel_weight is None else accel_weight,
                        None if "prev_qpos" in null else guards["prev_qpos"].ptr(),
                        None if "has_prev" in null else guards["has_prev"].ptr())
    err = C.create_string_buffer(600)
    rc = lib.emu_fixed_lag_step_accel(C.byref(table), C.byref(prm), C.byref(io), C.byref(acc),
                                      C.c_longlong(S if num_streams is None else num_streams),
                                      C.c_longlong(K if num_ticks is None else num_ticks), err, C.c_int(600))
    if rc != 0:
        raise EmulationError(rc, err.value.decode())
    for name, b in list(outs.items()) + list(guards.items()) + [("workspace", ws)]:
        b.check(name)
    for k, v in inputs.items():  # read-only inputs stay untouched
        if v is not None:
            np.testing.assert_array_equal(v, before[k], err_msg=f"{k} was written")
    for k, g in guards.items():
        state[k][...] = g.a
    return {k: g.a for k, g in outs.items()}


def smooth_pre_anchor(seq, keypoints, offsets, qpos_init, accel_weight, last_qpos, prev_qpos, has_prev, projected=None,
                      fixed_qpos=None, smooth_weight=-1.0):
    """smooth_packed_stream<G, true, true> on packed clips (emu_smooth_accel_host.smooth_packed's arguments, plus each
    stream's pre-anchor prev_qpos [S,n] and has_prev [S]).  Returns (qpos [N,n], robot_qpos [N,dof], status [N], cost [S])."""
    from dex_retargeting_b200 import _native as N

    lib = load()
    opt = seq.optimizer
    table = opt.build_table()
    prm = opt.params(clip_init=True, lp_alpha=seq.low_pass_alpha)
    f32 = (lambda a: None if a is None else np.ascontiguousarray(a, np.float32))
    kp = f32(keypoints).reshape(-1, N.NUM_KEYPOINTS, 3)
    offsets = np.ascontiguousarray(offsets, np.int64)
    S, Nf = len(offsets) - 1, kp.shape[0]
    inputs = dict(keypoints=kp, fixed_qpos=f32(fixed_qpos) if table.n_fixed else None, last_qpos=f32(last_qpos),
                  projected=None if projected is None else np.ascontiguousarray(projected, np.uint8),
                  qpos_init=f32(qpos_init))
    prev, has = f32(prev_qpos), np.ascontiguousarray(has_prev, np.int32)
    q = Guarded(np.full((Nf, table.n_var), np.nan, np.float32), np.float32(-7.0))
    rq = Guarded(np.full((Nf, table.dof), np.nan, np.float32), np.float32(-7.0))
    status = Guarded(np.full(Nf, -1, np.int32), np.int32(-9))
    cost = Guarded(np.full(S, np.nan, np.float32), np.float32(-7.0))
    nbytes = SA.workspace_bytes(seq, Nf)
    ws = Guarded(np.full(max(nbytes // 4, 1), np.nan, np.float32), np.float32(-7.0))
    io = N.DexrSmooth()
    for k, v in inputs.items():
        setattr(io, k, None if v is None else v.ctypes.data)
    io.qpos_out, io.robot_qpos_out, io.status_out, io.cost_out = q.ptr(), rq.ptr(), status.ptr(), cost.ptr()
    io.smooth_weight = smooth_weight
    io.workspace, io.workspace_bytes = ws.ptr(), nbytes
    pre = _accel_struct(accel_weight, prev.ctypes.data, has.ctypes.data)
    err = C.create_string_buffer(600)
    rc = lib.emu_smooth_packed_pre_anchor(C.byref(table), C.byref(prm), C.byref(io), C.byref(pre),
                                          C.c_void_p(offsets.ctypes.data), C.c_longlong(S), C.c_longlong(Nf), err,
                                          C.c_int(600))
    if rc != 0:
        raise EmulationError(rc, err.value.decode())
    for name, b in (("qpos_out", q), ("robot_qpos_out", rq), ("status_out", status), ("cost_out", cost), ("workspace", ws)):
        b.check(name)
    return q.a, rq.a, status.a, cost.a
