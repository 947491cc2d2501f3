#!/usr/bin/env python
"""Dry run of tests/test_gpu_fixed_lag_accel.py on the CPU, in the manner of tests/tools/emu_gpu_fixed_lag.py: the test
functions are called unchanged while SeqRetargeting.retarget_fixed_lag / flush_fixed_lag on an accelerated state are served
by the host emulation of the accelerated fixed-lag driver (tests/emu_fixed_lag_accel_host.py), smooth_packed_sequences by
the accel smoother's (tests/tools/emu_gpu_smooth_accel.py) and the causal calls by those of tests/tools/emu_gpu_packed.py.
The state tensors are CPU tensors whose memory the emulation updates in place.  The sizes are shrunk (STREAMS, CHECKED).
Not covered: the library's launch shape and shared-memory loop state, output views, the asynchrony of the call, GPU
arithmetic in the last bits (the GPU-against-emulation test compares the emulation with itself here).

  python tests/tools/emu_gpu_fixed_lag_accel.py [-k substring]
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
from dex_retargeting_b200.optimizer import Optimizer  # noqa: E402
from dex_retargeting_b200.seq_retarget import FixedLagTape, SeqRetargeting, _refuse_accel_backward  # noqa: E402

SKIP = {"test_calls_are_asynchronous": "needs a device stream",
        "test_writes_stay_inside_their_buffers": "needs device tensor views (the emulation guards every buffer itself)"}
SIZES = dict(STREAMS=3, CHECKED=2)


def _state_arrays(state):
    """The accelerated state as numpy arrays sharing the tensors' memory (the emulation writes them in place)."""
    d = {k: E._np(getattr(state, k)) for k in FA.STATE}
    d.update(lag=int(state.lag), accel_weight=float(state.accel_weight))
    return d


def retarget_fixed_lag(self, keypoints, state, *, fixed_qpos=None, smooth_weight=None, out=None, qpos_out=None,
                       status_out=None, stream=None, tape=None):
    _refuse_accel_backward(state, "retarget_fixed_lag(tape=...)", tape is not None)
    assert state.accel_weight, "the dry run serves accelerated states only"
    r = FA.fixed_lag_step(self, E._np(keypoints), _state_arrays(state), fixed_qpos=E._np(fixed_qpos),
                          smooth_weight=-1.0 if smooth_weight is None else smooth_weight)
    return FLG._put(out, r["robot_qpos"]), FLG._put(qpos_out, r["qpos"]), FLG._put(status_out, r["status"])


def flush_fixed_lag(self, state, *, out=None, qpos_out=None, count_out=None, stream=None):
    r = FA.fixed_lag_step(self, None, _state_arrays(state), flush=True)
    return FLG._put(out, r["flush_robot_qpos"]), FLG._put(qpos_out, r["flush_qpos"]), FLG._put(count_out, r["flush_count"])


def make_fixed_lag_tape(self, num_streams, num_ticks, lag):
    opt = self.optimizer
    lp = opt._objective_spec().len_proj
    return FixedLagTape(qpos=Q._from(np.zeros((num_streams, num_ticks, lag + 1, opt.opt_dof), np.float32)),
                        projected=Q._from(np.zeros((num_streams, num_ticks, lp), np.uint8)) if lp else None)


def main():
    Optimizer.engine = lambda self: E.FakeEngine(self)
    SeqRetargeting.make_stream_state = E.make_stream_state
    SeqRetargeting.make_sequence_tape = Q.make_sequence_tape
    SeqRetargeting.retarget_sequences = Q.retarget_sequences
    SeqRetargeting.pack_streams = K.pack_streams
    SeqRetargeting.make_packed_sequence_tape = K.make_packed_sequence_tape
    SeqRetargeting.retarget_packed_sequences = K.retarget_packed_sequences
    SeqRetargeting.smooth_packed_sequences = SAG.smooth_packed_sequences
    SeqRetargeting.retarget_fixed_lag = retarget_fixed_lag
    SeqRetargeting.flush_fixed_lag = flush_fixed_lag
    SeqRetargeting.make_fixed_lag_tape = make_fixed_lag_tape
    import test_gpu_fixed_lag_accel

    mod = test_gpu_fixed_lag_accel
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
