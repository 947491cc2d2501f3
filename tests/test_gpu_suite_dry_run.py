"""The GPU test functions, dry-run on the CPU: tests/tools/emu_gpu_tests.py calls the functions of tests/test_gpu_golden.py,
tests/test_gpu_arrow.py and tests/test_gpu_structures.py unchanged, with the device entry points of the host mirror served by the host emulation of the
solver source (tests/emu).  Run in a subprocess because the runner patches Optimizer / SeqRetargeting for its process.
Keeps the -m gpu tests and the solver source honest between GPU slots: a change that would turn them red shows up here."""
import subprocess
import sys
from pathlib import Path

import pytest

ROOT = Path(__file__).resolve().parent.parent


@pytest.mark.parametrize("subset,count", [("test_gpu_golden", 19), ("test_gpu_arrow", 11), ("test_gpu_structures", 33)])
def test_gpu_test_functions_pass_against_the_emulated_solver(subset, count):
    res = subprocess.run([sys.executable, str(ROOT / "tests" / "tools" / "emu_gpu_tests.py"), "-k", subset], capture_output=True,
                         text=True, timeout=900)
    tail = "\n".join(res.stdout.strip().splitlines()[-15:])
    assert res.returncode == 0 and f"{count}/{count} passed" in res.stdout, tail + res.stderr[-2000:]
