#!/usr/bin/env python
"""Dry run of tests/test_gpu_objective.py on the CPU, in the manner of tests/tools/emu_gpu_tests.py (whose torch proxy,
emulated retarget_batch and runner pieces it uses): the test functions are called unchanged while Optimizer.objective_batch
is served by the host emulation of the evaluation driver (tests/emu_eval_host.py) and Optimizer.retarget_batch by that of the
solver (tests/emu_host.py).  Not covered: the closure's own device buffers, the library's argument checks on a robot handle,
the 65 536-frame batch, GPU arithmetic in the last bits.

  python tests/tools/emu_gpu_objective.py [DEXR_EXP_FASTSINCOS] [-k substring]
"""
import sys
import tempfile
import time
import traceback
from pathlib import Path

import torch as real_torch

sys.path.insert(0, str(Path(__file__).resolve().parent))
import emu_gpu_tests as E  # noqa: E402  (puts the repository and tests/ on sys.path)
import emu_eval_host  # noqa: E402
from dex_retargeting_b200.optimizer import Optimizer  # noqa: E402

SKIP = {"test_reference_closure_values_through_get_objective_function": "the closure's own device buffers",
        "test_argument_errors_are_rejected_with_a_message": "library entry on a robot handle",
        "test_full_bench_batch": "65 536-frame batch"}


def objective_batch(self, qpos, ref_value=None, fixed_qpos=None, last_qpos=None, *, keypoints=None, projected=None, raw_hand=None,
                    loss_out=None, cost_out=None, grad_out=None, want_grad=True, stream=None):
    np_ = E._np  # (in place: a tensor shares its memory with the array, so the flags are updated in the caller's tensor)
    res = emu_eval_host.eval_objective(self, np_(qpos), keypoints=np_(keypoints), ref_value=np_(ref_value),
                                       fixed_qpos=np_(fixed_qpos), last_qpos=np_(last_qpos), projected=np_(projected),
                                       raw_hand=raw_hand, want_grad=want_grad or grad_out is not None, defines=E.DEFINES)
    outs = []
    for dst, src in zip((loss_out, cost_out, grad_out), res):
        if src is not None and dst is not None:
            dst.copy_(real_torch.from_numpy(src))
        outs.append(dst if dst is not None or src is None else real_torch.from_numpy(src))
    return tuple(outs)


def main():
    Optimizer.retarget_batch = E.retarget_batch
    Optimizer.objective_batch = objective_batch
    Optimizer.engine = lambda self: E.FakeEngine(self)
    import test_gpu_objective
    import test_gpu_parity

    test_gpu_parity.torch = E.TorchProxy()  # (its _dev and gpu_solve serve the objective tests)
    mod = test_gpu_objective
    mod.torch = E.TorchProxy()
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
    print(f"{ran - failed}/{ran} passed with defines {E.DEFINES or '(default)'}")
    return failed


if __name__ == "__main__":
    sys.exit(1 if main() else 0)
