#!/usr/bin/env python
"""Dry run of tests/test_gpu_smooth.py on the CPU, in the manner of tests/tools/emu_gpu_packed.py: the test functions are
called unchanged while SeqRetargeting.smooth_packed_sequences is served by the host emulation of the smoother
(tests/emu_smooth_host.py) and the causal calls it starts from by the emulations of tests/tools/emu_gpu_packed.py.  The sizes
are shrunk (STREAMS, LO, HI, CHECKED, NEIGHBOURS, RECT_SIZE): the emulation solves a few frames per second.  Not covered: the library's launch
shape, the asynchrony of the call, GPU arithmetic in the last bits.

  python tests/tools/emu_gpu_smooth.py [-k substring]
"""
import sys
import time
import traceback
from pathlib import Path

import numpy as np

sys.path.insert(0, str(Path(__file__).resolve().parent))
import emu_gpu_packed as K  # noqa: E402
import emu_gpu_seq_vjp as Q  # noqa: E402
import emu_gpu_tests as E  # noqa: E402  (puts the repository and tests/ on sys.path)
import emu_smooth_host as SM  # noqa: E402
from dex_retargeting_b200.optimizer import Optimizer  # noqa: E402
from dex_retargeting_b200.seq_retarget import SeqRetargeting  # noqa: E402

SKIP = {"test_call_is_asynchronous": "needs a device stream"}
SIZES = dict(STREAMS=6, LO=3, HI=6, CHECKED=2, NEIGHBOURS=(4, 2, 4), RECT_SIZE=(3, 3))


def smooth_packed_sequences(self, keypoints, layout, state=None, *, fixed_qpos=None, qpos_init=None, smooth_weight=None,
                            out=None, status_out=None, stream=None):
    np_ = E._np
    state = state if state is not None else self.make_stream_state(layout.num_streams)
    if qpos_init is None:  # as the product: the taped causal solve on a copy of the state
        from dex_retargeting_b200.seq_retarget import StreamState

        tape = self.make_packed_sequence_tape(layout)
        copy = StreamState(**{k: (None if getattr(state, k) is None else getattr(state, k).clone())
                              for k in StreamState._FIELDS})
        self.retarget_packed_sequences(keypoints, layout, copy, fixed_qpos=fixed_qpos, tape=tape)
        qpos_init = tape.qpos
    q, rq, status, _ = SM.smooth_packed(self, np_(keypoints), np_(layout.offsets), np_(qpos_init),
                                        last_qpos=np_(state.last_qpos), projected=np_(state.projected),
                                        fixed_qpos=np_(fixed_qpos), smooth_weight=-1.0 if smooth_weight is None else smooth_weight)
    return Q._from(rq.copy()), Q._from(q.copy()), Q._from(status.copy())


def main():
    Optimizer.engine = lambda self: E.FakeEngine(self)
    SeqRetargeting.make_stream_state = E.make_stream_state
    SeqRetargeting.make_sequence_tape = Q.make_sequence_tape
    SeqRetargeting.retarget_sequences = Q.retarget_sequences
    SeqRetargeting.pack_streams = K.pack_streams
    SeqRetargeting.make_packed_sequence_tape = K.make_packed_sequence_tape
    SeqRetargeting.retarget_packed_sequences = K.retarget_packed_sequences
    SeqRetargeting.smooth_packed_sequences = smooth_packed_sequences
    import test_gpu_smooth

    mod = test_gpu_smooth
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
