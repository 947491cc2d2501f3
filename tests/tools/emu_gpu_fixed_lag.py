#!/usr/bin/env python
"""Dry run of tests/test_gpu_fixed_lag.py on the CPU, in the manner of tests/tools/emu_gpu_smooth.py: the test functions
are called unchanged while SeqRetargeting.retarget_fixed_lag / flush_fixed_lag are served by the host emulation of the
fixed-lag driver (tests/emu_fixed_lag_host.py), smooth_packed_sequences by the smoother's (tests/tools/emu_gpu_smooth.py)
and the causal calls by those of tests/tools/emu_gpu_packed.py.  The state tensors are CPU tensors whose memory the
emulation updates in place.  The sizes are shrunk (STREAMS, CHECKED): the emulation solves a few windows per second.  Not
covered: the library's launch shape and shared-memory loop state, the asynchrony of the call, GPU arithmetic in the last
bits (the GPU-against-emulation test compares the emulation with itself here).

  python tests/tools/emu_gpu_fixed_lag.py [-k substring]
"""
import sys
import tempfile
import time
import traceback
from pathlib import Path

import numpy as np

sys.path.insert(0, str(Path(__file__).resolve().parent))
import emu_gpu_packed as K  # noqa: E402
import emu_gpu_seq_vjp as Q  # noqa: E402
import emu_gpu_smooth as SMG  # noqa: E402
import emu_gpu_tests as E  # noqa: E402  (puts the repository and tests/ on sys.path)
import emu_fixed_lag_host as FL  # noqa: E402
from dex_retargeting_b200.optimizer import Optimizer  # noqa: E402
from dex_retargeting_b200.seq_retarget import SeqRetargeting  # noqa: E402

SKIP = {"test_call_is_asynchronous": "needs a device stream"}
SIZES = dict(STREAMS=3, CHECKED=2)
STATE = ("last_qpos", "projected", "window_keypoints", "window_fixed_qpos", "window_qpos", "window_len")


def _state_arrays(state):
    """The state as numpy arrays sharing the tensors' memory (the emulation writes them in place)."""
    d = {k: E._np(getattr(state, k)) for k in STATE}
    d["lag"] = int(state.lag)
    return d


def _put(dst, src):
    if dst is None:
        return Q._from(src.copy())
    dst.copy_(Q._from(np.ascontiguousarray(src)))
    return dst


def retarget_fixed_lag(self, keypoints, state, *, fixed_qpos=None, smooth_weight=None, out=None, qpos_out=None,
                       status_out=None, stream=None):
    r = FL.fixed_lag_step(self, E._np(keypoints), _state_arrays(state), fixed_qpos=E._np(fixed_qpos),
                          smooth_weight=-1.0 if smooth_weight is None else smooth_weight)
    return _put(out, r["robot_qpos"]), _put(qpos_out, r["qpos"]), _put(status_out, r["status"])


def flush_fixed_lag(self, state, *, out=None, qpos_out=None, count_out=None, stream=None):
    r = FL.fixed_lag_step(self, None, _state_arrays(state), flush=True)
    return _put(out, r["flush_robot_qpos"]), _put(qpos_out, r["flush_qpos"]), _put(count_out, r["flush_count"])


def main():
    Optimizer.engine = lambda self: E.FakeEngine(self)
    SeqRetargeting.make_stream_state = E.make_stream_state
    SeqRetargeting.make_sequence_tape = Q.make_sequence_tape
    SeqRetargeting.retarget_sequences = Q.retarget_sequences
    SeqRetargeting.pack_streams = K.pack_streams
    SeqRetargeting.make_packed_sequence_tape = K.make_packed_sequence_tape
    SeqRetargeting.retarget_packed_sequences = K.retarget_packed_sequences
    SeqRetargeting.smooth_packed_sequences = SMG.smooth_packed_sequences
    SeqRetargeting.retarget_fixed_lag = retarget_fixed_lag
    SeqRetargeting.flush_fixed_lag = flush_fixed_lag
    import test_gpu_fixed_lag

    mod = test_gpu_fixed_lag
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
