#!/usr/bin/env python
"""Dry run of tests/test_gpu_vjp.py on the CPU, in the manner of tests/tools/emu_gpu_objective.py: the test functions are
called unchanged while Optimizer.retarget_batch_vjp is served by the host emulation of the VJP driver (tests/emu_vjp_host.py)
and Optimizer.retarget_batch by that of the solver (tests/emu_host.py).  Not covered: the library's argument checks on a
robot handle, the 65 536-frame batch, GPU arithmetic in the last bits.

  python tests/tools/emu_gpu_vjp.py [-k substring]
"""
import sys
import tempfile
import time
import traceback
from pathlib import Path

import torch as real_torch

sys.path.insert(0, str(Path(__file__).resolve().parent))
import emu_gpu_tests as E  # noqa: E402  (puts the repository and tests/ on sys.path)
import emu_vjp_host  # noqa: E402
from dex_retargeting_b200.optimizer import Optimizer  # noqa: E402

SKIP = {"test_argument_errors_are_rejected_with_a_message": "library entry on a robot handle",
        "test_full_bench_batch": "65 536-frame batch"}


def retarget_batch_vjp(self, grad_qpos, qpos, ref_value=None, fixed_qpos=None, last_qpos=None, *, keypoints=None,
                       projected=None, grad_keypoints_out=None, grad_ref_value_out=None, grad_fixed_qpos_out=None,
                       grad_last_qpos_out=None, status_out=None, stream=None):
    np_ = E._np
    g_t, g_f, g_l, status = emu_vjp_host.solve_vjp(self, np_(grad_qpos), np_(qpos), keypoints=np_(keypoints),
                                                    ref_value=np_(ref_value), fixed_qpos=np_(fixed_qpos),
                                                    last_qpos=np_(last_qpos), projected=np_(projected))
    if status_out is not None:
        status_out.copy_(real_torch.from_numpy(status))
    return tuple(None if a is None else real_torch.from_numpy(a) for a in (g_t, g_f, g_l))


def main():
    Optimizer.retarget_batch = E.retarget_batch
    Optimizer.retarget_batch_vjp = retarget_batch_vjp
    Optimizer.engine = lambda self: E.FakeEngine(self)
    import test_gpu_parity
    import test_gpu_vjp

    test_gpu_parity.torch = E.TorchProxy()
    mod = test_gpu_vjp
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
    print(f"{ran - failed}/{ran} passed")
    return failed


if __name__ == "__main__":
    sys.exit(1 if main() else 0)
