#!/usr/bin/env python
"""Dry run of tests/test_gpu_fixed_lag_accel_vjp.py on the CPU, in the manner of tests/tools/emu_gpu_fixed_lag_accel.py:
the test functions are called unchanged while SeqRetargeting's accelerated fixed-lag forward (with and without a tape),
flush and backward (retarget_fixed_lag_accel_vjp, flush_fixed_lag_accel_vjp) are served by the host emulation of the kernels'
code (tests/emu_fixed_lag_accel_host.py, tests/emu_fixed_lag_accel_vjp_host.py), the offline accel VJP by
tests/tools/emu_gpu_smooth_accel.py's and the causal calls by tests/tools/emu_gpu_packed.py's.  The public methods' own
argument checks run first, as on the device.  The state tensors are CPU tensors whose memory the emulation updates in
place.  The sizes are shrunk (STREAMS, CHECKED).  Not covered: the library's launch shape and shared-memory loop state,
output views, the asynchrony of the call, GPU arithmetic in the last bits (the GPU-against-emulation test compares the
emulation with itself here).

  python tests/tools/emu_gpu_fixed_lag_accel_vjp.py [-k substring]
"""
import sys
import tempfile
import time
import traceback
from pathlib import Path

import numpy as np

sys.path.insert(0, str(Path(__file__).resolve().parent))
import emu_gpu_fixed_lag as FLG  # noqa: E402
import emu_gpu_packed as K  # noqa: E402
import emu_gpu_seq_vjp as Q  # noqa: E402
import emu_gpu_smooth_accel as SAG  # noqa: E402
import emu_gpu_tests as E  # noqa: E402  (puts the repository and tests/ on sys.path)
import emu_fixed_lag_accel_host as FA  # noqa: E402
import emu_fixed_lag_accel_vjp_host as AV  # noqa: E402
from dex_retargeting_b200.optimizer import Optimizer  # noqa: E402
from dex_retargeting_b200.seq_retarget import FixedLagTape, SeqRetargeting, _check_tape_accel  # noqa: E402

SKIP = {"test_backward_is_asynchronous": "needs a device stream",
        "test_writes_stay_inside_their_buffers": "needs device tensor views (the emulation guards every buffer itself)"}
SIZES = dict(STREAMS=4, BATCH=2, CHECKED=2)


def _state_arrays(state):
    """The accelerated state as numpy arrays sharing the tensors' memory (the emulation writes them in place)."""
    d = {k: E._np(getattr(state, k)) for k in FA.STATE}
    d.update(lag=int(state.lag), accel_weight=float(state.accel_weight))
    return d


def retarget_fixed_lag(self, keypoints, state, *, fixed_qpos=None, smooth_weight=None, out=None, qpos_out=None,
                       status_out=None, stream=None, tape=None):
    _check_tape_accel(state, tape)  # (the method's own refusal)
    assert state.accel_weight, "the dry run serves accelerated states only"
    w = -1.0 if smooth_weight is None else smooth_weight
    if tape is None:
        r = FA.fixed_lag_step(self, E._np(keypoints), _state_arrays(state), fixed_qpos=E._np(fixed_qpos), smooth_weight=w)
    else:
        r = AV.fixed_lag_step_accel_tape(self, E._np(keypoints), _state_arrays(state), fixed_qpos=E._np(fixed_qpos),
                                         smooth_weight=w)
        E._np(tape.qpos)[...] = r["tape_qpos"]
        if tape.projected is not None:
            E._np(tape.projected)[...] = r["tape_projected"]
    return FLG._put(out, r["robot_qpos"]), FLG._put(qpos_out, r["qpos"]), FLG._put(status_out, r["status"])


def flush_fixed_lag(self, state, *, out=None, qpos_out=None, count_out=None, stream=None):
    r = FA.fixed_lag_step(self, None, _state_arrays(state), flush=True)
    return FLG._put(out, r["flush_robot_qpos"]), FLG._put(qpos_out, r["flush_qpos"]), FLG._put(count_out, r["flush_count"])


def make_fixed_lag_tape(self, num_streams, num_ticks, lag, accel_weight=None):
    opt = self.optimizer
    lp = opt._objective_spec().len_proj
    return FixedLagTape(qpos=Q._from(np.zeros((num_streams, num_ticks, lag + 1, opt.opt_dof), np.float32)),
                        projected=Q._from(np.zeros((num_streams, num_ticks, lp), np.uint8)) if lp else None,
                        accel_weight=0.0 if accel_weight is None else float(accel_weight))


_OUT = ("grad_last_qpos", "grad_window_keypoints", "grad_window_fixed_qpos", "grad_window_qpos")


def _vjp(self, keypoints, tape, state0, fixed_qpos, flushed, smooth_weight=-1.0, **g):
    s0 = {k: (None if getattr(state0, k) is None else E._np(getattr(state0, k)).copy()) for k in FA.STATE}
    s0.update(lag=int(state0.lag), accel_weight=float(state0.accel_weight))
    return AV.fixed_lag_accel_vjp(self, E._np(keypoints), s0, None if tape is None else E._np(tape.qpos),
                                  None if tape is None else E._np(tape.projected), fixed_qpos=E._np(fixed_qpos),
                                  flushed=flushed, smooth_weight=smooth_weight, **{k: E._np(v) for k, v in g.items()})


def _t(a, nf):
    return None if a is None or (a.ndim >= 1 and a.shape[-1] == 0 and nf == 0) else Q._from(np.ascontiguousarray(a))


def retarget_fixed_lag_accel_vjp(self, keypoints, tape, state0, *, fixed_qpos=None, smooth_weight=None, stream=None,
                                 outputs=None, **g):
    self._accel_state0(state0, "retarget_fixed_lag_accel_vjp", tape)
    r = _vjp(self, keypoints, tape, state0, fixed_qpos, False,
             smooth_weight=-1.0 if smooth_weight is None else smooth_weight, **g)
    nf = len(self.optimizer.idx_pin2fixed)
    return (Q._from(r["grad_keypoints"]), _t(r["grad_fixed_qpos"], nf), *(_t(r[k], nf) for k in _OUT),
            Q._from(r["status"]), Q._from(r["grad_prev_qpos"]))


def flush_fixed_lag_accel_vjp(self, state0, *, grad_qpos=None, grad_robot_qpos=None, stream=None, **g):
    self._accel_state0(state0, "flush_fixed_lag_accel_vjp")
    r = _vjp(self, None, None, state0, None, True, grad_flush_qpos=grad_qpos, grad_flush_robot_qpos=grad_robot_qpos, **g)
    nf = len(self.optimizer.idx_pin2fixed)
    return (*(_t(r[k], nf) for k in _OUT), Q._from(r["grad_prev_qpos"]))


def main():
    Optimizer.engine = lambda self: E.FakeEngine(self)
    SeqRetargeting.make_stream_state = E.make_stream_state
    SeqRetargeting.pack_streams = K.pack_streams
    SeqRetargeting.make_packed_sequence_tape = K.make_packed_sequence_tape
    SeqRetargeting.retarget_packed_sequences = K.retarget_packed_sequences
    SeqRetargeting.smooth_packed_sequences_vjp = SAG.smooth_packed_sequences_vjp
    SeqRetargeting.retarget_fixed_lag = retarget_fixed_lag
    SeqRetargeting.flush_fixed_lag = flush_fixed_lag
    SeqRetargeting.make_fixed_lag_tape = make_fixed_lag_tape
    SeqRetargeting.retarget_fixed_lag_accel_vjp = retarget_fixed_lag_accel_vjp
    SeqRetargeting.flush_fixed_lag_accel_vjp = flush_fixed_lag_accel_vjp
    import test_gpu_fixed_lag_accel_vjp

    mod = test_gpu_fixed_lag_accel_vjp
    mod.torch = E.TorchProxy()
    for k, v in SIZES.items():
        setattr(mod, k, v)
    failed = ran = 0
    for name in [n for n in dir(mod) if n.startswith("test_")]:
        fn = getattr(mod, name)
        if name in SKIP:
            print(f"SKIP {name}: {SKIP[name]}")
            continue
        for kw in E.expand(fn):
            label = f"{mod.__name__}::{name} {kw if kw else ''}"
            if E.KEYWORD and E.KEYWORD not in label:
                continue
            if "tmp_path" in fn.__code__.co_varnames[:fn.__code__.co_argcount]:
                kw = dict(kw, tmp_path=Path(tempfile.mkdtemp()))
            t0 = time.time()
            ran += 1
            try:
                fn(**kw)
                print(f"PASS {label} [{time.time() - t0:.1f}s]", flush=True)
            except Exception:
                failed += 1
                print(f"FAIL {label}\n{traceback.format_exc(limit=6)}", flush=True)
    print(f"{ran - failed}/{ran} passed")
    return failed


if __name__ == "__main__":
    np.seterr(all="ignore")
    sys.exit(1 if main() else 0)
