#!/usr/bin/env python
"""Dry run of the GPU parity suite on the CPU: the test functions of tests/test_gpu_{parity,golden,arrow,structures,newton_step}.py are called
unchanged while the two device entry points of the host mirror (Optimizer.retarget_batch, SeqRetargeting.retarget_sequences)
are served by the HOST EMULATION of the solver source (tests/emu) -- for a chosen set of compile-time experiment switches.
Inside the test modules `torch` is a proxy that maps every device to the CPU.  Not covered: the pinned-host entry, multi-GPU,
anything that is specific to the kernels of dexr.cu (tile ring, alignment paths), GPU arithmetic in the last bits.

  python tests/tools/emu_gpu_tests.py                                   # default build of the solver
  python tests/tools/emu_gpu_tests.py DEXR_EXP_PDFALLBACK DEXR_EXP_FKNOISE [-k substring]
"""
import itertools
import os
import sys
import tempfile
import time
import traceback
from pathlib import Path

import numpy as np
import torch as real_torch

ROOT = Path(__file__).resolve().parents[2]
for p in (ROOT, ROOT / "tests"):
    sys.path.insert(0, str(p))
import emu_host  # noqa: E402
from dex_retargeting_b200.optimizer import Optimizer  # noqa: E402
from dex_retargeting_b200.seq_retarget import SeqRetargeting, StreamState  # noqa: E402

ARGS = sys.argv[1:]
KEYWORD = ARGS[ARGS.index("-k") + 1] if "-k" in ARGS else None
DEFINES = tuple(a for a in ARGS if a.startswith("DEXR_EXP_"))
SKIP = {"test_host_buffer_entry_matches_device_entry": "pinned-host entry (dexr_solve_frames_host)",
        "test_batch_shapes_alignment_and_determinism": "alignment / tile paths of the CUDA kernel",
        "test_full_batch_properties": "65 536-frame batch (hours under emulation)",
        "test_single_frame_api_matches_batch_and_oracle": "single-frame host entry",
        "test_maximum_size_robot_parity": "uses the host entry",
        "test_empty_batch_is_a_no_op": "host entry",
        "test_carried_damping_through_every_entry_point": "host entries (the device part passes: 0.95 of the cold starts in the same minimum)",
        "test_mixed_launch_with_structure_cases": "mixed-robot launch (dexr_solve_frames_multi)"}


class FakeEngine:
    """Stands in for optimizer._Engine (which creates the device copy of the table): only launch_info is asked for."""

    def __init__(self, opt):
        t = opt.build_table()
        self.lanes = 16 if t.dof <= 16 else 32

    def launch_info(self):
        return dict(grid=1, block=32, smem_bytes=0, frames_per_tile=32 // self.lanes, lanes_per_frame=self.lanes,
                    consumer_warps=1, kernels_launched=0)


class _Cuda:
    synchronize = staticmethod(lambda *a, **k: None)
    is_available = staticmethod(lambda: True)
    device_count = staticmethod(lambda: 1)


class TorchProxy:
    cuda = _Cuda()

    def device(self, *a, **k):
        return real_torch.device("cpu")

    def __getattr__(self, name):
        return getattr(real_torch, name)


def _np(t):
    return None if t is None else t.detach().numpy()


def use_arrow():
    return os.environ.get("DEXR_ARROW", "1") != "0"


def retarget_batch(self, ref_value=None, fixed_qpos=None, last_qpos=None, *, keypoints=None, projected=None, out=None,
                   robot_qpos_out=None, status_out=None, cost_out=None, clip_init=False, stream=None, damping=None):
    B = last_qpos.shape[0]
    if B == 0:
        return real_torch.empty((0, self.opt_dof)) if out is None else out
    q, status, cost, full = emu_host.solve_frames(self, _np(last_qpos), keypoints=_np(keypoints), ref_value=_np(ref_value),
                                                 fixed_qpos=_np(fixed_qpos), projected=_np(projected), defines=DEFINES,
                                                 use_arrow=use_arrow(), clip_init=clip_init, want_robot_qpos=True,
                                                 damping=_np(damping))  # (in place: the tensor shares its memory with the array)
    for dst, src in ((status_out, status), (cost_out, cost), (robot_qpos_out, full)):
        if dst is not None:
            dst.copy_(real_torch.from_numpy(src))
    if out is not None:
        out.copy_(real_torch.from_numpy(q))
        return out
    return real_torch.from_numpy(q)


def make_stream_state(self, num_streams):
    opt = self.optimizer
    lp = opt._objective_spec().len_proj
    return StreamState(last_qpos=real_torch.from_numpy(np.tile(self.joint_limits.mean(1).astype(np.float32), (num_streams, 1))),
                       filter_state=real_torch.zeros((num_streams, opt.robot.dof)), filter_init=real_torch.zeros(num_streams, dtype=real_torch.uint8),
                       projected=real_torch.zeros((num_streams, lp), dtype=real_torch.uint8) if lp else None,
                       damping=real_torch.zeros(num_streams))


def retarget_sequences(self, keypoints, state=None, fixed_qpos=None, out=None, status_out=None, stream=None):
    S = keypoints.shape[0]
    state = state if state is not None else self.make_stream_state(S)
    st = dict(last_qpos=_np(state.last_qpos), filter_state=_np(state.filter_state), filter_init=_np(state.filter_init),
              projected=_np(state.projected), damping=_np(state.damping))
    # DEXR_SEQ_DUO=1: the scarce-streams mode of the 16-lane solver (the library's choice for few streams unless set to 0)
    got, status, _ = emu_host.solve_sequences(self, _np(keypoints), state=st, defines=DEFINES, use_arrow=use_arrow(),
                                              fixed_qpos=_np(fixed_qpos), duo=os.environ.get("DEXR_SEQ_DUO") == "1")
    if status_out is not None:
        status_out.copy_(real_torch.from_numpy(status))
    if out is not None:
        out.copy_(real_torch.from_numpy(got))
        return out, state
    return real_torch.from_numpy(got), state


class EnvPatch:
    """Stand-in for pytest's monkeypatch (setenv / delenv only; the emulated entry points ignore the library's switches)."""

    def setenv(self, k, v):
        os.environ[k] = v

    def delenv(self, k, raising=True):
        os.environ.pop(k, None)


def expand(fn):
    marks = [m for m in getattr(fn, "pytestmark", []) if m.name == "parametrize"]
    axes = []
    for m in marks:
        names = [n.strip() for n in m.args[0].split(",")]
        axes.append([dict(zip(names, v if len(names) > 1 else (v,))) for v in m.args[1]])
    for combo in itertools.product(*axes) if axes else [()]:
        kw = {}
        for d in combo:
            kw.update(d)
        yield kw


def main():
    Optimizer.retarget_batch = retarget_batch
    Optimizer.engine = lambda self: FakeEngine(self)
    SeqRetargeting.make_stream_state = make_stream_state
    SeqRetargeting.retarget_sequences = retarget_sequences
    import test_gpu_arrow, test_gpu_golden, test_gpu_newton_step, test_gpu_parity, test_gpu_structures  # noqa: E401

    failed = ran = 0
    for mod in (test_gpu_parity, test_gpu_golden, test_gpu_arrow, test_gpu_structures, test_gpu_newton_step):
        mod.torch = TorchProxy()
        for name in [n for n in dir(mod) if n.startswith("test_")]:
            fn = getattr(mod, name)
            if name in SKIP:
                print(f"SKIP {name}: {SKIP[name]}")
                continue
            for kw in expand(fn):
                label = f"{mod.__name__}::{name} {kw if kw else ''}"
                if KEYWORD and KEYWORD not in label:
                    continue
                if "tmp_path" in fn.__code__.co_varnames[:fn.__code__.co_argcount]:
                    kw = dict(kw, tmp_path=Path(tempfile.mkdtemp()))
                if "monkeypatch" in fn.__code__.co_varnames[:fn.__code__.co_argcount]:
                    kw = dict(kw, monkeypatch=EnvPatch())
                t0 = time.time()
                ran += 1
                try:
                    fn(**kw)
                    print(f"PASS {label} [{time.time() - t0:.1f}s]", flush=True)
                except Exception:
                    failed += 1
                    print(f"FAIL {label}\n{traceback.format_exc(limit=4)}", flush=True)
    print(f"{ran - failed}/{ran} passed with defines {DEFINES or '(default)'}")
    return failed


if __name__ == "__main__":
    sys.exit(1 if main() else 0)
