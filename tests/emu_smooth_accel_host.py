"""Host emulation of the acceleration-penalised smoother and its backpropagation (TEST INFRASTRUCTURE): builds
tests/emu/emu_smooth_accel.cpp -- the fiber-warp emulation of tests/emu/emu_driver.cpp plus smooth_packed_stream<G, true>
and smooth_vjp_packed_stream<G, true> of dex_retargeting_b200/csrc/dexr_kernels.cuh -- with g++ and calls
emu_smooth_sequences_packed_accel(_vjp) through ctypes.  Every buffer the driver may write lies between guard words,
checked after each call, and the inputs must come back unchanged.  Used by tests/test_smooth_accel_emulation.py and
tests/tools/emu_gpu_smooth_accel.py; never by the product."""
import ctypes as C
import subprocess
from functools import lru_cache

import numpy as np

from emu_eval_host import EMU, ROOT, EmulationError, _out_dir
from emu_packed_host import Guarded

SOURCES = [EMU / "emu_smooth_accel.cpp", EMU / "emu_driver.cpp", EMU / "warp_shim.h",
           ROOT / "dex_retargeting_b200" / "csrc" / "dexr_kernels.cuh", ROOT / "include" / "dexr.h"]


@lru_cache(maxsize=None)
def load():
    so = _out_dir() / "libdexr_emu_smooth_accel.so"
    if not so.exists() or any(so.stat().st_mtime < p.stat().st_mtime for p in SOURCES):
        # -O0 as for emu_driver.cpp: the rendezvous protocol compares the call sites of the lanes
        cmd = ["g++", "-O0", "-std=c++17", "-fPIC", "-shared", f"-I{EMU / 'stub'}", "-o", str(so),
               str(EMU / "emu_smooth_accel.cpp")]
        res = subprocess.run(cmd, capture_output=True, text=True)
        if res.returncode != 0:
            raise RuntimeError("g++ failed building the host emulation:\n" + res.stderr[-4000:])
    lib = C.CDLL(str(so))
    lib.emu_smooth_sequences_packed_accel.restype = C.c_int
    lib.emu_smooth_sequences_packed_accel_vjp.restype = C.c_int
    lib.emu_smooth_accel_workspace_bytes.restype = C.c_size_t
    return lib


def workspace_bytes(seq, num_frames):
    return int(load().emu_smooth_accel_workspace_bytes(C.byref(seq.optimizer.build_table()), C.c_longlong(num_frames)))


def _f32(a):
    return None if a is None else np.ascontiguousarray(a, dtype=np.float32)


def smooth_packed(seq, keypoints, offsets, qpos_init, accel_weight, last_qpos=None, projected=None, fixed_qpos=None,
                  smooth_weight=-1.0, num_streams=None, null=(), workspace_bytes=None, params=None):
    """Emulated dexr_smooth_sequences_packed_accel (arguments as emu_smooth_host.smooth_packed, plus accel_weight).
    Returns (qpos [N,n], robot_qpos [N,dof], status [N], cost [S])."""
    from dex_retargeting_b200 import _native as N

    lib = load()
    opt = seq.optimizer
    table = opt.build_table()
    prm = opt.params(clip_init=True, lp_alpha=seq.low_pass_alpha) if params is None else params
    kp = _f32(keypoints).reshape(-1, N.NUM_KEYPOINTS, 3)
    offsets = np.ascontiguousarray(offsets, np.int64)
    S = len(offsets) - 1 if num_streams is None else num_streams
    Nf = kp.shape[0]
    inputs = dict(keypoints=kp, fixed_qpos=_f32(fixed_qpos) if table.n_fixed else None, last_qpos=_f32(last_qpos),
                  projected=None if projected is None else np.ascontiguousarray(projected, np.uint8),
                  qpos_init=_f32(qpos_init))
    before = {k: None if v is None else v.copy() for k, v in inputs.items()}
    q = Guarded(np.full((Nf, table.n_var), np.nan, np.float32), np.float32(-7.0))
    rq = Guarded(np.full((Nf, table.dof), np.nan, np.float32), np.float32(-7.0))
    status = Guarded(np.full(Nf, -1, np.int32), np.int32(-9))
    cost = Guarded(np.full(max(S, 0), np.nan, np.float32), np.float32(-7.0))
    nbytes = int(lib.emu_smooth_accel_workspace_bytes(C.byref(table), C.c_longlong(Nf))) if workspace_bytes is None \
        else workspace_bytes
    ws = Guarded(np.full(max(nbytes // 4, 1), np.nan, np.float32), np.float32(-7.0))
    io = N.DexrSmooth()
    for k, v in inputs.items():
        setattr(io, k, None if v is None or k in null else v.ctypes.data)
    io.qpos_out = None if "qpos_out" in null else q.ptr()
    io.robot_qpos_out = None if "robot_qpos_out" in null else rq.ptr()
    io.status_out = None if "status_out" in null else status.ptr()
    io.cost_out = None if "cost_out" in null else cost.ptr()
    io.smooth_weight = smooth_weight
    io.workspace = None if "workspace" in null else ws.ptr()
    io.workspace_bytes = nbytes
    err = C.create_string_buffer(600)
    rc = lib.emu_smooth_sequences_packed_accel(C.byref(table), C.byref(prm), C.byref(io), C.c_float(accel_weight),
                                               C.c_void_p(None if "offsets" in null else offsets.ctypes.data),
                                               C.c_longlong(S), C.c_longlong(Nf), err, C.c_int(600))
    if rc != 0:
        raise EmulationError(rc, err.value.decode())
    for name, b in (("qpos_out", q), ("robot_qpos_out", rq), ("status_out", status), ("cost_out", cost), ("workspace", ws)):
        b.check(name)
    for k, v in inputs.items():  # read-only inputs stay untouched
        if v is not None:
            np.testing.assert_array_equal(v, before[k], err_msg=f"{k} was written")
    return q.a, rq.a, status.a, cost.a


def smooth_vjp_packed(seq, keypoints, offsets, qpos, accel_weight, last_qpos=None, projected=None, fixed_qpos=None,
                      grad_qpos=None, grad_robot_qpos=None, smooth_weight=-1.0, num_streams=None, null=(),
                      workspace_bytes=None, params=None):
    """Emulated dexr_smooth_sequences_packed_accel_vjp (arguments as emu_smooth_vjp_host.smooth_vjp_packed, plus
    accel_weight).  Returns (grad_keypoints [N,21,3], grad_fixed [N,n_fixed], grad_last [S,n] or None, status [N])."""
    from dex_retargeting_b200 import _native as N

    lib = load()
    opt = seq.optimizer
    table = opt.build_table()
    prm = opt.params(clip_init=True, lp_alpha=seq.low_pass_alpha) if params is None else params
    kp = _f32(keypoints).reshape(-1, N.NUM_KEYPOINTS, 3)
    offsets = np.ascontiguousarray(offsets, np.int64)
    S = len(offsets) - 1 if num_streams is None else num_streams
    Nf = kp.shape[0]
    inputs = dict(keypoints=kp, fixed_qpos=_f32(fixed_qpos) if table.n_fixed else None, last_qpos=_f32(last_qpos),
                  projected=None if projected is None else np.ascontiguousarray(projected, np.uint8), qpos=_f32(qpos),
                  grad_qpos=_f32(grad_qpos), grad_robot_qpos=_f32(grad_robot_qpos))
    before = {k: None if v is None else v.copy() for k, v in inputs.items()}
    gk = Guarded(np.full((Nf, N.NUM_KEYPOINTS, 3), np.nan, np.float32), np.float32(-7.0))
    gf = Guarded(np.full((Nf, table.n_fixed), np.nan, np.float32), np.float32(-7.0))
    gl = Guarded(np.full((max(S, 0), table.n_var), np.nan, np.float32), np.float32(-7.0))
    status = Guarded(np.full(Nf, -1, np.int32), np.int32(-9))
    nbytes = int(lib.emu_smooth_accel_workspace_bytes(C.byref(table), C.c_longlong(Nf))) if workspace_bytes is None \
        else workspace_bytes
    ws = Guarded(np.full(max(nbytes // 4, 1), np.nan, np.float32), np.float32(-7.0))
    io = N.DexrSmoothVjp()
    for k, v in inputs.items():
        setattr(io, k, None if v is None or k in null else v.ctypes.data)
    io.grad_keypoints = None if "grad_keypoints" in null else gk.ptr()
    io.grad_fixed_qpos = None if "grad_fixed_qpos" in null or table.n_fixed == 0 else gf.ptr()
    io.grad_last_qpos = None if "grad_last_qpos" in null or last_qpos is None else gl.ptr()
    io.status_out = None if "status_out" in null else status.ptr()
    io.smooth_weight = smooth_weight
    io.workspace = None if "workspace" in null else ws.ptr()
    io.workspace_bytes = nbytes
    err = C.create_string_buffer(600)
    rc = lib.emu_smooth_sequences_packed_accel_vjp(C.byref(table), C.byref(prm), C.byref(io), C.c_float(accel_weight),
                                                   C.c_void_p(None if "offsets" in null else offsets.ctypes.data),
                                                   C.c_longlong(S), C.c_longlong(Nf), err, C.c_int(600))
    if rc != 0:
        raise EmulationError(rc, err.value.decode())
    for name, b in (("grad_keypoints", gk), ("grad_fixed_qpos", gf), ("grad_last_qpos", gl), ("status_out", status),
                    ("workspace", ws)):
        b.check(name)
    for k, v in inputs.items():  # read-only inputs stay untouched
        if v is not None:
            np.testing.assert_array_equal(v, before[k], err_msg=f"{k} was written")
    return gk.a, gf.a, (gl.a if last_qpos is not None else None), status.a
