#!/usr/bin/env python
"""Dry run of tests/test_gpu_seq_vjp.py on the CPU, in the manner of tests/tools/emu_gpu_vjp.py: the test functions are
called unchanged while SeqRetargeting.retarget_sequences (recorded or not) and retarget_sequences_vjp are served by the host
emulation of the stream drivers (tests/emu_host.py, tests/emu_seq_vjp_host.py) and Optimizer.retarget_batch_vjp by that of
the VJP driver (tests/emu_vjp_host.py).  The recorded-forward and per-frame-loop checks run at FORWARD_SIZE / LOOP_SIZE
shrunk to a few streams and frames (the emulation solves a few frames per second).  Not covered: the library's argument
checks on a robot handle, the library's launch shapes, GPU arithmetic in the last bits.

  python tests/tools/emu_gpu_seq_vjp.py [-k substring]
"""
import sys
import tempfile
import time
import traceback
from pathlib import Path

import torch as real_torch

sys.path.insert(0, str(Path(__file__).resolve().parent))
import emu_gpu_tests as E  # noqa: E402  (puts the repository and tests/ on sys.path)
import emu_gpu_vjp  # noqa: E402
import emu_host  # noqa: E402
import emu_seq_vjp_host as H  # noqa: E402
from dex_retargeting_b200.optimizer import Optimizer  # noqa: E402
from dex_retargeting_b200.seq_retarget import SeqRetargeting, SequenceTape  # noqa: E402

SKIP = {"test_argument_errors_are_rejected_with_a_message": "library entry on a robot handle"}
SIZES = dict(FORWARD_SIZE=(6, 5), LOOP_SIZE=(6, 4))


def _from(a):
    return None if a is None else real_torch.from_numpy(a)


def make_sequence_tape(self, num_streams, num_steps):
    opt = self.optimizer
    lp = opt._objective_spec().len_proj
    return SequenceTape(qpos=real_torch.empty((num_streams, num_steps, opt.opt_dof)),
                        projected=(real_torch.empty((num_streams, num_steps, lp), dtype=real_torch.uint8)
                                   if opt.retargeting_type == "DEXPILOT" else None))


def retarget_sequences(self, keypoints, state=None, fixed_qpos=None, out=None, status_out=None, stream=None, raw_hand=None,
                       tape=None):
    np_ = E._np
    state = state if state is not None else self.make_stream_state(keypoints.shape[0])
    st = dict(last_qpos=np_(state.last_qpos), filter_state=np_(state.filter_state), filter_init=np_(state.filter_init),
              projected=np_(state.projected), damping=np_(state.damping))  # (views: the state is updated in place)
    if tape is None:
        got, status, _ = emu_host.solve_sequences(self, np_(keypoints), state=st, use_arrow=E.use_arrow(),
                                                  fixed_qpos=np_(fixed_qpos))
    else:
        got, status, _, tp = H.solve_sequences_tape(self, np_(keypoints), state=st, fixed_qpos=np_(fixed_qpos),
                                                    use_arrow=E.use_arrow())
        tape.qpos.copy_(_from(tp["qpos"]))
        if tape.projected is not None:
            tape.projected.copy_(_from(tp["projected"]))
    if status_out is not None:
        status_out.copy_(_from(status))
    if out is not None:
        out.copy_(_from(got))
        return out, state
    return _from(got), state


def retarget_sequences_vjp(self, keypoints, tape, last_qpos0, filter_init0, grad_robot_qpos=None, grad_last_qpos=None,
                           grad_filter_state=None, fixed_qpos=None, grad_keypoints_out=None, grad_fixed_qpos_out=None,
                           grad_last_qpos_out=None, grad_filter_state_out=None, status_out=None, stream=None):
    np_ = E._np
    g_kp, g_fixed, g_last, g_filter, status = H.solve_sequences_vjp(
        self, np_(keypoints), np_(tape.qpos), np_(last_qpos0), np_(filter_init0), np_(tape.projected),
        grad_robot_qpos=np_(grad_robot_qpos), grad_last_qpos=np_(grad_last_qpos), grad_filter_state=np_(grad_filter_state),
        fixed_qpos=np_(fixed_qpos))
    if status_out is not None:
        status_out.copy_(_from(status))
    return _from(g_kp), _from(g_fixed), _from(g_last), _from(g_filter)


def main():
    Optimizer.retarget_batch = E.retarget_batch
    Optimizer.retarget_batch_vjp = emu_gpu_vjp.retarget_batch_vjp
    Optimizer.engine = lambda self: E.FakeEngine(self)
    SeqRetargeting.make_stream_state = E.make_stream_state
    SeqRetargeting.make_sequence_tape = make_sequence_tape
    SeqRetargeting.retarget_sequences = retarget_sequences
    SeqRetargeting.retarget_sequences_vjp = retarget_sequences_vjp
    import test_gpu_seq_vjp

    mod = test_gpu_seq_vjp
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
