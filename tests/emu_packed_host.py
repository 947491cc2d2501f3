"""Host emulation of packed streams (TEST INFRASTRUCTURE): builds tests/emu/emu_packed.cpp -- the fiber-warp emulation of
tests/emu/emu_driver.cpp plus the packed-stream drivers of dex_retargeting_b200/csrc/dexr_kernels.cuh -- with g++ and calls
emu_solve_sequences_packed / emu_solve_sequences_packed_vjp through ctypes.  Every buffer the drivers may write lies between
guard words, checked after each call: a layout must never make them write outside their buffers.  Used by
tests/test_packed_streams_emulation.py and tests/tools/emu_gpu_packed.py; never by the product."""
import ctypes as C
import subprocess
from functools import lru_cache

import numpy as np

from emu_eval_host import EMU, ROOT, EmulationError, _out_dir
from emu_seq_vjp_host import fresh_state

SOURCES = [EMU / "emu_packed.cpp", EMU / "emu_driver.cpp", EMU / "warp_shim.h",
           ROOT / "dex_retargeting_b200" / "csrc" / "dexr_kernels.cuh", ROOT / "include" / "dexr.h"]
GUARD = 16  # guard elements on each side of every written buffer


@lru_cache(maxsize=None)
def load():
    so = _out_dir() / "libdexr_emu_packed.so"
    if not so.exists() or any(so.stat().st_mtime < p.stat().st_mtime for p in SOURCES):
        # -O0 as for emu_driver.cpp: the rendezvous protocol compares the call sites of the lanes
        cmd = ["g++", "-O0", "-std=c++17", "-fPIC", "-shared", f"-I{EMU / 'stub'}", "-o", str(so), str(EMU / "emu_packed.cpp")]
        res = subprocess.run(cmd, capture_output=True, text=True)
        if res.returncode != 0:
            raise RuntimeError("g++ failed building the host emulation:\n" + res.stderr[-4000:])
    lib = C.CDLL(str(so))
    lib.emu_solve_sequences_packed.restype = C.c_int
    lib.emu_solve_sequences_packed_vjp.restype = C.c_int
    return lib


class Guarded:
    """A buffer with GUARD sentinel elements on each side: `.a` is the buffer, `.check()` asserts the guards are intact."""

    def __init__(self, a, sentinel):
        a = np.ascontiguousarray(a)
        self.full = np.full(a.size + 2 * GUARD, sentinel, a.dtype)
        self.a = self.full[GUARD:GUARD + a.size].reshape(a.shape)
        self.a[...] = a
        self.sentinel = sentinel

    def ptr(self):
        return self.a.ctypes.data

    def check(self, name):
        for part in (self.full[:GUARD], self.full[GUARD + self.a.size:]):
            assert np.array_equal(part.view(np.uint8), np.full(part.shape, self.sentinel, part.dtype).view(np.uint8)), \
                f"{name}: a guard word outside the buffer was written"


def offsets_of(lengths):
    return np.concatenate([[0], np.cumsum(np.asarray(lengths, np.int64))]).astype(np.int64)


def _f32(a):
    return None if a is None else np.ascontiguousarray(a, dtype=np.float32)


def _ptr(a):
    return None if a is None else a.ctypes.data


def solve_packed(seq, keypoints, offsets, state=None, fixed_qpos=None, record=False, duo=False, use_arrow=True,
                 raw_hand=None, num_streams=None, null=()):
    """Emulated dexr_solve_sequences_packed: keypoints [N,21,3], offsets [S+1] (as given: malformed layouts included).
    Returns (robot_qpos [N,dof], status [N], state, tape) with tape = dict(qpos [N,n], projected [N,len_proj] or None) or
    None; `state` (numpy dict, emu_seq_vjp_host.fresh_state) is updated in place.  Outputs start as NaN / -1 / 7."""
    from dex_retargeting_b200 import _native as N

    lib = load()
    opt = seq.optimizer
    table, prm = opt.build_table(), opt.params(clip_init=True, lp_alpha=seq.low_pass_alpha, raw_hand=raw_hand)
    kp = _f32(keypoints).reshape(-1, N.NUM_KEYPOINTS, 3)
    offsets = np.ascontiguousarray(offsets, np.int64)
    S = len(offsets) - 1 if num_streams is None else num_streams
    Nf = kp.shape[0]
    state = fresh_state(seq, max(S, 0)) if state is None else state
    g = {k: Guarded(v, 0xAB if v.dtype == np.uint8 else np.nan) for k, v in state.items() if v is not None}
    out = Guarded(np.full((Nf, table.dof), np.nan, np.float32), np.float32(-7.0))
    status = Guarded(np.full(Nf, -1, np.int32), np.int32(-9))
    tq = tp = None
    if record:
        tq = Guarded(np.full((Nf, table.n_var), np.nan, np.float32), np.float32(-7.0))
        if opt.retargeting_type == "DEXPILOT":
            tp = Guarded(np.full((Nf, table.len_proj), 7, np.uint8), np.uint8(0xAB))
    io = N.DexrSequences()
    io.keypoints = None if "keypoints" in null else _ptr(kp)
    io.fixed_qpos = None if table.n_fixed == 0 or "fixed_qpos" in null else _ptr(_f32(fixed_qpos))
    for k, f in (("last_qpos", "last_qpos"), ("filter_state", "filter_state"), ("filter_init", "filter_init"),
                 ("projected", "projected"), ("damping", "damping_state")):
        setattr(io, f, None if k not in g or k in null else g[k].ptr())
    io.robot_qpos_out, io.status_out = out.ptr(), status.ptr()
    tape = N.DexrSequencesTape()
    if record:
        tape.qpos = None if "tape_qpos" in null else tq.ptr()
        tape.projected = None if tp is None or "tape_projected" in null else tp.ptr()
    err = C.create_string_buffer(600)
    rc = lib.emu_solve_sequences_packed(C.byref(table), C.byref(prm), C.c_int(int(use_arrow)), C.byref(io),
                                        C.byref(tape) if record else None, C.c_void_p(None if "offsets" in null else _ptr(offsets)),
                                        C.c_longlong(S), C.c_longlong(Nf), C.c_int(int(duo)), err,
                                        C.c_int(600))
    if rc != 0:
        raise EmulationError(rc, err.value.decode())
    for k, v in g.items():
        v.check(k)
        state[k][...] = v.a
    for name, b in (("robot_qpos_out", out), ("status_out", status), ("tape.qpos", tq), ("tape.projected", tp)):
        if b is not None:
            b.check(name)
    tape_out = None if not record else dict(qpos=tq.a, projected=None if tp is None else tp.a)
    return out.a, status.a, state, tape_out


def solve_packed_vjp(seq, keypoints, offsets, tape_qpos, last_qpos0, filter_init0=None, tape_projected=None,
                     grad_robot_qpos=None, grad_last_qpos=None, grad_filter_state=None, fixed_qpos=None, spw=0,
                     num_streams=None, null=(), raw_hand=None):
    """Emulated dexr_solve_sequences_packed_vjp.  Returns (grad_keypoints [N,21,3], grad_fixed [N,n_fixed] or None,
    grad_last_qpos0 [S,n], grad_filter_state0 [S,dof], status [N]); outputs start as NaN / -1, guard words around them."""
    from dex_retargeting_b200 import _native as N

    lib = load()
    opt = seq.optimizer
    table, prm = opt.build_table(), opt.params(clip_init=True, lp_alpha=seq.low_pass_alpha, raw_hand=raw_hand)
    kp = _f32(keypoints).reshape(-1, N.NUM_KEYPOINTS, 3)
    offsets = np.ascontiguousarray(offsets, np.int64)
    S = len(offsets) - 1 if num_streams is None else num_streams
    Nf = kp.shape[0]
    arrays = dict(keypoints=kp, fixed_qpos=_f32(fixed_qpos) if table.n_fixed > 0 else None, last_qpos=_f32(last_qpos0),
                  filter_init=None if filter_init0 is None else np.ascontiguousarray(filter_init0, np.uint8),
                  qpos=_f32(tape_qpos), projected=None if tape_projected is None else np.ascontiguousarray(tape_projected, np.uint8),
                  grad_robot_qpos=_f32(grad_robot_qpos), grad_last_qpos_out=_f32(grad_last_qpos),
                  grad_filter_state_out=_f32(grad_filter_state))
    g_kp = Guarded(np.full((Nf, N.NUM_KEYPOINTS, 3), np.nan, np.float32), np.float32(-7.0))
    g_fixed = Guarded(np.full((Nf, table.n_fixed), np.nan, np.float32), np.float32(-7.0)) if table.n_fixed else None
    g_last = Guarded(np.full((max(S, 0), table.n_var), np.nan, np.float32), np.float32(-7.0))
    g_filter = Guarded(np.full((max(S, 0), table.dof), np.nan, np.float32), np.float32(-7.0))
    status = Guarded(np.full(Nf, -1, np.int32), np.int32(-9))
    io = N.DexrSequencesVjp()
    for k, a in arrays.items():
        setattr(io, k, None if k in null else _ptr(a))
    io.grad_keypoints, io.grad_last_qpos, io.grad_filter_state = g_kp.ptr(), g_last.ptr(), g_filter.ptr()
    io.grad_fixed_qpos = None if g_fixed is None else g_fixed.ptr()
    io.status_out = status.ptr()
    err = C.create_string_buffer(600)
    rc = lib.emu_solve_sequences_packed_vjp(C.byref(table), C.byref(prm), C.byref(io),
                                            C.c_void_p(None if "offsets" in null else _ptr(offsets)), C.c_longlong(S), C.c_longlong(Nf), C.c_int(int(spw)), err, C.c_int(600))
    if rc != 0:
        raise EmulationError(rc, err.value.decode())
    for name, b in (("grad_keypoints", g_kp), ("grad_fixed_qpos", g_fixed), ("grad_last_qpos", g_last),
                    ("grad_filter_state", g_filter), ("status_out", status)):
        if b is not None:
            b.check(name)
    return g_kp.a, None if g_fixed is None else g_fixed.a, g_last.a, g_filter.a, status.a
