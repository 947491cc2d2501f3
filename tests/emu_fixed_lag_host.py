"""Host emulation of fixed-lag smoothing (TEST INFRASTRUCTURE): builds tests/emu/emu_fixed_lag.cpp -- the fiber-warp
emulation of tests/emu/emu_driver.cpp plus fixed_lag_tick of dex_retargeting_b200/csrc/dexr_kernels.cuh -- with g++ and
calls emu_fixed_lag_step through ctypes.  Every buffer the driver may write, the stream state included, lies between guard
words, checked after each call.  Used by tests/test_fixed_lag_emulation.py and tests/tools/emu_gpu_fixed_lag.py; never by
the product."""
import ctypes as C
import subprocess
from functools import lru_cache

import numpy as np

from emu_eval_host import EMU, ROOT, EmulationError, _out_dir
from emu_packed_host import Guarded

SOURCES = [EMU / "emu_fixed_lag.cpp", EMU / "emu_driver.cpp", EMU / "warp_shim.h",
           ROOT / "dex_retargeting_b200" / "csrc" / "dexr_kernels.cuh", ROOT / "include" / "dexr.h"]
STATE = ("last_qpos", "projected", "window_keypoints", "window_fixed_qpos", "window_qpos", "window_len")


@lru_cache(maxsize=None)
def load():
    so = _out_dir() / "libdexr_emu_fixed_lag.so"
    if not so.exists() or any(so.stat().st_mtime < p.stat().st_mtime for p in SOURCES):
        # -O0 as for emu_driver.cpp: the rendezvous protocol compares the call sites of the lanes
        cmd = ["g++", "-O0", "-std=c++17", "-fPIC", "-shared", f"-I{EMU / 'stub'}", "-o", str(so),
               str(EMU / "emu_fixed_lag.cpp")]
        res = subprocess.run(cmd, capture_output=True, text=True)
        if res.returncode != 0:
            raise RuntimeError("g++ failed building the host emulation:\n" + res.stderr[-4000:])
    lib = C.CDLL(str(so))
    lib.emu_fixed_lag_step.restype = C.c_int
    lib.emu_fixed_lag_workspace_bytes.restype = C.c_size_t
    return lib


def workspace_bytes(seq, S, lag):
    return int(load().emu_fixed_lag_workspace_bytes(C.byref(seq.optimizer.build_table()), C.c_longlong(S), C.c_int(lag)))


def fresh_state(seq, S, lag):
    """SeqRetargeting.make_fixed_lag_state as numpy arrays (plus "lag")."""
    opt = seq.optimizer
    table = opt.build_table()
    return dict(lag=int(lag), last_qpos=np.tile(seq.joint_limits.mean(1).astype(np.float32), (S, 1)),
                projected=np.zeros((S, table.len_proj), np.uint8) if table.len_proj else None,
                window_keypoints=np.zeros((S, lag + 1, 21, 3), np.float32),
                window_fixed_qpos=np.zeros((S, lag + 1, table.n_fixed), np.float32) if table.n_fixed else None,
                window_qpos=np.zeros((S, lag + 1, table.n_var), np.float32), window_len=np.zeros(S, np.int32))


def copy_state(st):
    return {k: (v.copy() if isinstance(v, np.ndarray) else v) for k, v in st.items()}


def fixed_lag_step(seq, keypoints, state, fixed_qpos=None, smooth_weight=-1.0, flush=False, null=(), workspace_bytes=None,
                   params=None, num_streams=None, num_ticks=None, lag=None):
    """Emulated dexr_fixed_lag_step: keypoints [S,K,21,3] (None: K = 0), fixed_qpos [S,K,n_fixed], `state` a numpy dict
    (`fresh_state`), updated in place.  Returns dict(qpos [S,K,n], robot_qpos [S,K,dof], status [S,K], and with `flush`
    flush_qpos [S,L,n], flush_robot_qpos [S,L,dof], flush_count [S]); every output starts filled (NaN, -3 or -1) inside
    guard words.  `params`: a dexr_params_t (default: the optimizer's)."""
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
    nbytes = int(lib.emu_fixed_lag_workspace_bytes(C.byref(table), C.c_longlong(S), C.c_int(L))) \
        if workspace_bytes is None else workspace_bytes
    ws = Guarded(np.full(max(nbytes // 4, 1), np.nan, np.float32), np.float32(-7.0))
    io = N.DexrFixedLag()
    for k, v in inputs.items():
        setattr(io, k, None if v is None or k in null else v.ctypes.data)
    for k, g in guards.items():
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
    err = C.create_string_buffer(600)
    rc = lib.emu_fixed_lag_step(C.byref(table), C.byref(prm), C.byref(io), C.c_longlong(S if num_streams is None else num_streams),
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
