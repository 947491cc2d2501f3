"""Register budget of the block-diagonal frames kernel (`dexr_frames_kernel<16, 4, NCW>`, the headline).

Its speed follows how much it spills at the register cap of its warp count (DESIGN.md section 3.1): the spill stores that
ptxas reports for the 24- and 28-warp builds must stay within what the kernel reaches today.  The `-Xptxas -v` lines
come from the library's build log when it is current, otherwise from a build of the same sources with the same flags
under a temporary directory (the tree may be read-only).
"""
import re
import shutil
import subprocess
from pathlib import Path

import pytest

from dex_retargeting_b200 import build as B

# consumer warps -> spill stores (bytes) allowed for dexr_frames_kernel<16, 4, consumer warps>
BUDGET = {23: 96, 27: 176}


def ptxas_log(tmp_path: Path) -> str:
    log = B.PKG / "csrc" / "build.log"
    if log.exists() and B.OUT.exists() and all(log.stat().st_mtime >= d.stat().st_mtime for d in B.DEPS):
        text = log.read_text()
        if "spill stores" in text:
            return text
    res = subprocess.run([B.find_nvcc(), *B.NVCC_FLAGS, "-o", str(tmp_path / "libdexr.so"), str(B.SRC)],
                         capture_output=True, text=True)
    assert res.returncode == 0, res.stderr[-2000:]
    return res.stdout + res.stderr


def spill_stores(log: str) -> dict:
    """mangled kernel name -> spill store bytes, from `-Xptxas -v` output"""
    out = {}
    for m in re.finditer(r"Function properties for (\S+)\n\s*\d+ bytes stack frame, (\d+) bytes spill stores", log):
        out[m.group(1)] = int(m.group(2))
    return out


@pytest.mark.skipif(shutil.which("nvcc") is None and not Path("/usr/local/cuda/bin/nvcc").exists(), reason="needs nvcc")
def test_block_frames_kernel_spill_budget(tmp_path):
    stores = spill_stores(ptxas_log(tmp_path))
    for ncw, budget in BUDGET.items():
        name = f"_ZN4dexr18dexr_frames_kernelILi16ELi4ELi{ncw}EEEvNS_9FrameArgsE"
        assert name in stores, f"no ptxas line for dexr_frames_kernel<16, 4, {ncw}>"
        assert stores[name] <= budget, (
            f"dexr_frames_kernel<16, 4, {ncw}> ({ncw + 1} warps per SM) spills {stores[name]} B of stores, budget {budget} B: "
            f"the block solver's live state grew (see DESIGN.md section 3.1 for where its register peaks are)")
