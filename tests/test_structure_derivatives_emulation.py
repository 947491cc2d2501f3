"""tests/test_gpu_structure_derivatives.py dry-run on the CPU (tests/tools/emu_gpu_structure_derivatives.py): the evaluation,
VJP, Jacobian, sequence-VJP, packed-stream and smoothing tests on the synthetic robots of tests/structure_cases.py, with every
entry point served by the host emulation of its driver.  The GPU-against-emulation comparisons are not run here."""
import subprocess
import sys
from pathlib import Path

ROOT = Path(__file__).resolve().parent.parent


def test_gpu_structure_derivatives_file_passes_against_the_emulation():
    count = 136
    res = subprocess.run([sys.executable, str(ROOT / "tests" / "tools" / "emu_gpu_structure_derivatives.py")],
                         capture_output=True, text=True, timeout=3600)
    tail = "\n".join(res.stdout.strip().splitlines()[-15:])
    assert res.returncode == 0 and f"{count}/{count} passed" in res.stdout, tail + res.stderr[-2000:]
