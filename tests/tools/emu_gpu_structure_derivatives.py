#!/usr/bin/env python
"""Dry run of tests/test_gpu_structure_derivatives.py on the CPU: the test functions are called unchanged while every entry
point they use is served by the host emulation of its driver, through the patches of tests/tools/emu_gpu_objective.py,
emu_gpu_vjp.py, emu_gpu_jacobian.py, emu_gpu_seq_vjp.py, emu_gpu_packed.py and emu_gpu_smooth.py, at the GPU file's own
sizes.  The comparisons of the GPU against the host emulation are skipped (they would compare the emulation with itself).
Not covered: the library's launch shapes, GPU arithmetic in the last bits.

  python tests/tools/emu_gpu_structure_derivatives.py [-k substring]
"""
import sys
import tempfile
import time
import traceback
from pathlib import Path

import numpy as np

sys.path.insert(0, str(Path(__file__).resolve().parent))
import emu_gpu_jacobian  # noqa: E402
import emu_gpu_objective  # noqa: E402
import emu_gpu_packed as K  # noqa: E402
import emu_gpu_seq_vjp as Q  # noqa: E402
import emu_gpu_smooth  # noqa: E402
import emu_gpu_tests as E  # noqa: E402  (puts the repository and tests/ on sys.path)
import emu_gpu_vjp  # noqa: E402
from dex_retargeting_b200.optimizer import Optimizer  # noqa: E402
from dex_retargeting_b200.seq_retarget import SeqRetargeting  # noqa: E402

SKIP = {"test_objective_matches_the_host_emulation": "GPU against the emulation",
        "test_vjp_matches_the_host_emulation": "GPU against the emulation"}


def main():
    Optimizer.retarget_batch = E.retarget_batch
    Optimizer.objective_batch = emu_gpu_objective.objective_batch
    Optimizer.retarget_batch_vjp = emu_gpu_vjp.retarget_batch_vjp
    Optimizer.retarget_batch_jacobian = emu_gpu_jacobian.retarget_batch_jacobian
    Optimizer.engine = lambda self: E.FakeEngine(self)
    SeqRetargeting.make_stream_state = E.make_stream_state
    SeqRetargeting.make_sequence_tape = Q.make_sequence_tape
    SeqRetargeting.retarget_sequences = Q.retarget_sequences
    SeqRetargeting.retarget_sequences_vjp = Q.retarget_sequences_vjp
    SeqRetargeting.pack_streams = K.pack_streams
    SeqRetargeting.make_packed_sequence_tape = K.make_packed_sequence_tape
    SeqRetargeting.retarget_packed_sequences = K.retarget_packed_sequences
    SeqRetargeting.retarget_packed_sequences_vjp = K.retarget_packed_sequences_vjp
    SeqRetargeting.smooth_packed_sequences = emu_gpu_smooth.smooth_packed_sequences
    import test_gpu_jacobian
    import test_gpu_objective
    import test_gpu_packed_streams
    import test_gpu_parity
    import test_gpu_smooth
    import test_gpu_structure_derivatives
    import test_gpu_vjp

    for m in (test_gpu_parity, test_gpu_objective, test_gpu_vjp, test_gpu_jacobian, test_gpu_packed_streams, test_gpu_smooth,
              test_gpu_structure_derivatives):
        m.torch = E.TorchProxy()  # (the helpers the new file imports run in their own modules)
    mod = test_gpu_structure_derivatives
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
            args = fn.__code__.co_varnames[:fn.__code__.co_argcount]
            if "tmp_path" in args:
                kw = dict(kw, tmp_path=Path(tempfile.mkdtemp()))
            env = E.EnvPatch()
            if "monkeypatch" in args:
                kw = dict(kw, monkeypatch=env)
            t0 = time.time()
            ran += 1
            try:
                fn(**kw)
                print(f"PASS {label} [{time.time() - t0:.1f}s]", flush=True)
            except Exception:
                failed += 1
                print(f"FAIL {label}\n{traceback.format_exc(limit=4)}", flush=True)
            finally:
                env.delenv("DEXR_SEQ_DUO", raising=False)
    print(f"{ran - failed}/{ran} passed")
    return failed


if __name__ == "__main__":
    np.seterr(all="ignore")
    sys.exit(1 if main() else 0)
