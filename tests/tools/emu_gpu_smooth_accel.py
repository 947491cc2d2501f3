#!/usr/bin/env python
"""Dry run of tests/test_gpu_smooth_accel.py on the CPU, in the manner of tests/tools/emu_gpu_smooth_vjp.py: the test
functions are called unchanged while SeqRetargeting.smooth_packed_sequences and smooth_packed_sequences_vjp are served by the
host emulation of the acceleration-penalised smoother and its VJP (tests/emu_smooth_accel_host.py; accel_weight None or 0:
the velocity-only emulations, as the library delegates) and the causal calls by the emulations of
tests/tools/emu_gpu_packed.py.  The sizes are shrunk (STREAMS, LO, HI, CHECKED, NEIGHBOURS).  Not covered: the library's
launch shape, autograd, output views, the asynchrony of the calls, GPU arithmetic in the last bits.

  python tests/tools/emu_gpu_smooth_accel.py [-k substring]
"""
import inspect
import sys
import tempfile
import time
import traceback
from pathlib import Path

import numpy as np

sys.path.insert(0, str(Path(__file__).resolve().parent))
import emu_gpu_packed as K  # noqa: E402
import emu_gpu_seq_vjp as Q  # noqa: E402
import emu_gpu_tests as E  # noqa: E402  (puts the repository and tests/ on sys.path)
import emu_smooth_accel_host as AH  # noqa: E402
import emu_smooth_host as SM  # noqa: E402
import emu_smooth_vjp_host as SVH  # noqa: E402
from dex_retargeting_b200.optimizer import Optimizer  # noqa: E402
from dex_retargeting_b200.seq_retarget import SeqRetargeting  # noqa: E402

SKIP = {"test_calls_are_asynchronous": "needs a device stream",
        "test_autograd_is_the_direct_call": "needs torch autograd on device tensors",
        "test_writes_stay_inside_their_buffers": "needs device tensor views (the emulation guards every buffer itself)",
        "test_gpu_matches_the_emulation": "compares the device with this emulation"}
SIZES = dict(STREAMS=3, LO=3, HI=5, CHECKED=2, NEIGHBOURS=(4, 2, 4))


def smooth_packed_sequences(self, keypoints, layout, state=None, *, fixed_qpos=None, qpos_init=None, smooth_weight=None,
                            accel_weight=None, out=None, status_out=None, stream=None):
    np_ = E._np
    state = state if state is not None else self.make_stream_state(layout.num_streams)
    if qpos_init is None:  # as the product: the taped causal solve on a copy of the state
        from dex_retargeting_b200.seq_retarget import StreamState

        tape = self.make_packed_sequence_tape(layout)
        copy = StreamState(**{k: (None if getattr(state, k) is None else getattr(state, k).clone())
                              for k in StreamState._FIELDS})
        self.retarget_packed_sequences(keypoints, layout, copy, fixed_qpos=fixed_qpos, tape=tape)
        qpos_init = tape.qpos
    kw = dict(last_qpos=np_(state.last_qpos), projected=np_(state.projected), fixed_qpos=np_(fixed_qpos),
              smooth_weight=-1.0 if smooth_weight is None else smooth_weight)
    c = 0.0 if accel_weight is None else float(accel_weight)
    args = (self, np_(keypoints), np_(layout.offsets), np_(qpos_init))
    q, rq, status, _ = AH.smooth_packed(*args, c, **kw) if c != 0.0 else SM.smooth_packed(*args, **kw)
    return Q._from(rq.copy()), Q._from(q.copy()), Q._from(status.copy())


def smooth_packed_sequences_vjp(self, keypoints, layout, qpos, last_qpos0=None, projected0=None, grad_qpos=None,
                                grad_robot_qpos=None, *, fixed_qpos=None, smooth_weight=None, accel_weight=None,
                                grad_keypoints_out=None, grad_fixed_qpos_out=None, grad_last_qpos_out=None, status_out=None,
                                stream=None):
    np_ = E._np
    kw = dict(last_qpos=np_(last_qpos0), projected=np_(projected0), fixed_qpos=np_(fixed_qpos), grad_qpos=np_(grad_qpos),
              grad_robot_qpos=np_(grad_robot_qpos), smooth_weight=-1.0 if smooth_weight is None else smooth_weight)
    c = 0.0 if accel_weight is None else float(accel_weight)
    args = (self, np_(keypoints), np_(layout.offsets), np_(qpos))
    g_kp, g_f, g_l, st = AH.smooth_vjp_packed(*args, c, **kw) if c != 0.0 else SVH.smooth_vjp_packed(*args, **kw)
    if status_out is not None:
        np_(status_out)[...] = st
    return Q._from(g_kp.copy()), (Q._from(g_f.copy()) if g_f.size else None), \
        (None if g_l is None else Q._from(g_l.copy()))


def main():
    Optimizer.engine = lambda self: E.FakeEngine(self)
    SeqRetargeting.make_stream_state = E.make_stream_state
    SeqRetargeting.make_sequence_tape = Q.make_sequence_tape
    SeqRetargeting.retarget_sequences = Q.retarget_sequences
    SeqRetargeting.pack_streams = K.pack_streams
    SeqRetargeting.make_packed_sequence_tape = K.make_packed_sequence_tape
    SeqRetargeting.retarget_packed_sequences = K.retarget_packed_sequences
    SeqRetargeting.smooth_packed_sequences = smooth_packed_sequences
    SeqRetargeting.smooth_packed_sequences_vjp = smooth_packed_sequences_vjp
    import test_gpu_smooth_accel

    mod = test_gpu_smooth_accel
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
            t0 = time.time()
            ran += 1
            try:
                if "tmp_path" in inspect.signature(fn).parameters:
                    kw = dict(kw, tmp_path=Path(tempfile.mkdtemp()))
                fn(**kw)
                print(f"PASS {label} [{time.time() - t0:.1f}s]", flush=True)
            except Exception:
                failed += 1
                print(f"FAIL {label}\n{traceback.format_exc(limit=4)}", flush=True)
    print(f"{ran - failed}/{ran} passed")
    return failed


if __name__ == "__main__":
    np.seterr(all="ignore")
    sys.exit(1 if main() else 0)
