#!/usr/bin/env python
"""Dry run of tests/test_gpu_jacobian.py on the CPU, in the manner of tests/tools/emu_gpu_vjp.py: the test functions are
called unchanged while Optimizer.retarget_batch_jacobian is served by the host emulation of the Jacobian driver
(tests/emu_jacobian_host.py), Optimizer.retarget_batch_vjp by that of the VJP driver and Optimizer.retarget_batch by that of
the solver (tests/emu_host.py).  Not covered: the library's argument checks on a robot handle, the 65 536-frame batch, GPU
arithmetic in the last bits.

  python tests/tools/emu_gpu_jacobian.py [-k substring]
"""
import sys
import tempfile
import time
import traceback
from pathlib import Path

import torch as real_torch

sys.path.insert(0, str(Path(__file__).resolve().parent))
import emu_gpu_tests as E  # noqa: E402  (puts the repository and tests/ on sys.path)
import emu_jacobian_host  # noqa: E402
from emu_gpu_vjp import retarget_batch_vjp  # noqa: E402
from dex_retargeting_b200.optimizer import Optimizer  # noqa: E402

SKIP = {"test_argument_errors_are_rejected_with_a_message": "library entry on a robot handle",
        "test_full_bench_batch": "65 536-frame batch"}


def retarget_batch_jacobian(self, qpos, ref_value=None, fixed_qpos=None, last_qpos=None, *, keypoints=None, projected=None,
                            jac_keypoints_out=None, jac_ref_value_out=None, jac_fixed_qpos_out=None, jac_last_qpos_out=None,
                            status_out=None, stream=None):
    np_ = E._np
    j_t, j_f, j_l, status = emu_jacobian_host.solve_jacobian(self, np_(qpos), keypoints=np_(keypoints),
                                                             ref_value=np_(ref_value), fixed_qpos=np_(fixed_qpos),
                                                             last_qpos=np_(last_qpos), projected=np_(projected))
    if status_out is not None:
        status_out.copy_(real_torch.from_numpy(status))
    return tuple(None if a is None else real_torch.from_numpy(a) for a in (j_t, j_f, j_l))


def main():
    Optimizer.retarget_batch = E.retarget_batch
    Optimizer.retarget_batch_vjp = retarget_batch_vjp
    Optimizer.retarget_batch_jacobian = retarget_batch_jacobian
    Optimizer.engine = lambda self: E.FakeEngine(self)
    import test_gpu_jacobian
    import test_gpu_parity

    test_gpu_parity.torch = E.TorchProxy()
    mod = test_gpu_jacobian
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
