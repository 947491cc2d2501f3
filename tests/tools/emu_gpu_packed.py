#!/usr/bin/env python
"""Dry run of tests/test_gpu_packed_streams.py on the CPU, in the manner of tests/tools/emu_gpu_seq_vjp.py: the test
functions are called unchanged while SeqRetargeting's packed calls (retarget_packed_sequences, recorded or not, and
retarget_packed_sequences_vjp) are served by the host emulation of the packed-stream drivers (tests/emu_packed_host.py) and
the rectangular ones by that of the stream drivers (tests/emu_host.py, tests/emu_seq_vjp_host.py).  The sizes are shrunk
(EQUAL_SIZE, RAGGED_STREAMS): the emulation solves a few frames per second.  Not covered: the library's argument checks on a
robot handle, the library's launch shapes, the benchmark's 2048-stream workloads, GPU arithmetic in the last bits.

  python tests/tools/emu_gpu_packed.py [-k substring]
"""
import sys
import tempfile
import time
import traceback
from pathlib import Path

import numpy as np
import torch as real_torch

sys.path.insert(0, str(Path(__file__).resolve().parent))
import emu_gpu_seq_vjp as Q  # noqa: E402
import emu_gpu_tests as E  # noqa: E402  (puts the repository and tests/ on sys.path)
import emu_packed_host as P  # noqa: E402
from dex_retargeting_b200.optimizer import Optimizer  # noqa: E402
from dex_retargeting_b200.seq_retarget import PackedStreams, SeqRetargeting, SequenceTape  # noqa: E402

SKIP = {"test_argument_errors_are_rejected_with_a_message": "library entry on a robot handle",
        "test_ragged_workloads_match_the_oracle": "the benchmark's 2048-stream workloads (hours under emulation)"}
SIZES = dict(EQUAL_SIZE=(3, 3), RAGGED_STREAMS=6, RAGGED_CHECKED=6)


def pack_streams(self, lengths):
    lens = np.asarray(lengths)
    if lens.ndim != 1 or (lens.size and not np.issubdtype(lens.dtype, np.integer)) or (lens < 0).any():
        raise ValueError("stream lengths must be >= 0")
    lens = lens.astype(np.int64)
    return PackedStreams(lengths=tuple(int(v) for v in lens), offsets=real_torch.from_numpy(P.offsets_of(lens)))


def make_packed_sequence_tape(self, layout):
    opt = self.optimizer
    lp = opt._objective_spec().len_proj
    return SequenceTape(qpos=real_torch.empty((layout.num_frames, opt.opt_dof)),
                        projected=(real_torch.empty((layout.num_frames, lp), dtype=real_torch.uint8)
                                   if opt.retargeting_type == "DEXPILOT" else None))


def retarget_packed_sequences(self, keypoints, layout, state=None, fixed_qpos=None, out=None, status_out=None, stream=None,
                              raw_hand=None, tape=None):
    np_ = E._np
    state = state if state is not None else self.make_stream_state(layout.num_streams)
    st = dict(last_qpos=np_(state.last_qpos), filter_state=np_(state.filter_state), filter_init=np_(state.filter_init),
              projected=np_(state.projected), damping=np_(state.damping))  # (views: the state is updated in place)
    got, status, _, tp = P.solve_packed(self, np_(keypoints), np_(layout.offsets), state=st, fixed_qpos=np_(fixed_qpos),
                                        record=tape is not None, use_arrow=E.use_arrow(),
                                        raw_hand=raw_hand)
    if tape is not None:
        tape.qpos.copy_(Q._from(tp["qpos"]))
        if tape.projected is not None:
            tape.projected.copy_(Q._from(tp["projected"]))
    if status_out is not None:
        status_out.copy_(Q._from(status))
    if out is not None:
        out.copy_(Q._from(got))
        return out, state
    return Q._from(got.copy()), state


def retarget_packed_sequences_vjp(self, keypoints, layout, tape, last_qpos0, filter_init0, grad_robot_qpos=None,
                                  grad_last_qpos=None, grad_filter_state=None, fixed_qpos=None, grad_keypoints_out=None,
                                  grad_fixed_qpos_out=None, grad_last_qpos_out=None, grad_filter_state_out=None,
                                  status_out=None, stream=None):
    np_ = E._np
    g_kp, g_fixed, g_last, g_filter, status = P.solve_packed_vjp(
        self, np_(keypoints), np_(layout.offsets), np_(tape.qpos), np_(last_qpos0), np_(filter_init0), np_(tape.projected),
        grad_robot_qpos=np_(grad_robot_qpos), grad_last_qpos=np_(grad_last_qpos), grad_filter_state=np_(grad_filter_state),
        fixed_qpos=np_(fixed_qpos))
    if layout.num_frames == 0:
        g_last[...] = 0 if grad_last_qpos is None else np_(grad_last_qpos)
        g_filter[...] = 0 if grad_filter_state is None else np_(grad_filter_state)
    if status_out is not None:
        status_out.copy_(Q._from(status))
    c = (lambda a: None if a is None else Q._from(a.copy()))
    return c(g_kp), c(g_fixed), c(g_last), c(g_filter)


def main():
    Optimizer.engine = lambda self: E.FakeEngine(self)
    SeqRetargeting.make_stream_state = E.make_stream_state
    SeqRetargeting.make_sequence_tape = Q.make_sequence_tape
    SeqRetargeting.retarget_sequences = Q.retarget_sequences
    SeqRetargeting.retarget_sequences_vjp = Q.retarget_sequences_vjp
    SeqRetargeting.pack_streams = pack_streams
    SeqRetargeting.make_packed_sequence_tape = make_packed_sequence_tape
    SeqRetargeting.retarget_packed_sequences = retarget_packed_sequences
    SeqRetargeting.retarget_packed_sequences_vjp = retarget_packed_sequences_vjp
    import test_gpu_packed_streams

    mod = test_gpu_packed_streams
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
                print(f"FAIL {label}\n{traceback.format_exc(limit=4)}", flush=True)
    print(f"{ran - failed}/{ran} passed")
    return failed


if __name__ == "__main__":
    sys.exit(1 if main() else 0)
