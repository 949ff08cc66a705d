"""Compile-time guard of the splat rasteriser's local-memory use (no GPU needed: nvcc cross-compiles for sm_90a).

k_splat_project runs ~41 M fragments per 640x480 frame of the -static workload through its fragment loop.  While the IEEE divisions of
the exact path sat inside that loop, their slow-path calls made ptxas spill around every unit and every round (120 B of spill stores,
144 B of spill loads), and the spills went to L2.  The exact path now runs from a per-warp queue outside the loop; this test reads what
the compiler made of the kernel under the shipped flags."""
import os
import re
import shutil
import subprocess

import pytest

from maskfusion_b200 import build as B

KERNEL = "_ZN3mfb15k_splat_projectEPK6float4S2_S2_PKjPKNS_7DevPoseENS_3CamEiifffffjS2_Py"
SRC = os.path.join(B.CSRC, "mf_surfel.cu")

pytestmark = pytest.mark.skipif(not shutil.which(B.NVCC) and not os.path.exists(B.NVCC), reason="nvcc not available")


def test_splat_kernel_does_not_spill(tmp_path):
    cmd = [B.NVCC] + B.ARCH + B.COMMON + B.SOURCES["mf_surfel.cu"] + ["-I", B.CSRC, "-c", "-o", str(tmp_path / "mf_surfel.o"), "-Xptxas", "-v", SRC]
    r = subprocess.run(cmd, capture_output=True, text=True, cwd=tmp_path)
    assert r.returncode == 0, r.stderr[-3000:]
    m = re.search(r"Function properties for " + re.escape(KERNEL) + r"\s*\n\s*(\d+) bytes stack frame, (\d+) bytes spill stores, (\d+) bytes spill loads",
                  r.stderr)
    assert m, r.stderr[-3000:]
    stores, loads = int(m.group(2)), int(m.group(3))
    assert stores == 0 and loads == 0, f"k_splat_project spills: {stores} B of stores, {loads} B of loads"
