"""Compile-time checks of the persistent tracker's normal equations on the fp64 tensor core (no GPU needed: nvcc cross-compiles for sm_90a).

Each warp sums the outer products of its pixels' rows with mma.m8n8k4.f64 instead of keeping 29 fp64 accumulators per thread across the
pixel loop; with the per-thread accumulators the kernel spilled 230 bytes of registers under its 128-register cap.  These tests read what
the compiler made of k_track_persistent with the shipped flags."""
import os
import re
import shutil
import subprocess

import pytest

from maskfusion_b200 import build as B

KERNEL = "_ZN3mfb18k_track_persistentEPKNS_8TrackJobENS_11TrackParamsE"
SRC = os.path.join(B.CSRC, "mf_track.cu")
CUOBJDUMP = os.path.join(os.path.dirname(B.NVCC), "cuobjdump")
# what remains are per-level values reloaded outside the pixel loops; the per-thread accumulators spilled 230 / 388 bytes
MAX_SPILL_BYTES = 32

pytestmark = pytest.mark.skipif(not shutil.which(B.NVCC) and not os.path.exists(B.NVCC), reason="nvcc not available")


def _compile(tmp_path):
    obj = tmp_path / "mf_track.o"
    cmd = [B.NVCC] + B.ARCH + B.COMMON + B.SOURCES["mf_track.cu"] + ["-I", B.CSRC, "-c", "-o", str(obj), "-Xptxas", "-v", SRC]
    r = subprocess.run(cmd, capture_output=True, text=True, cwd=tmp_path)
    assert r.returncode == 0, r.stderr[-3000:]
    return obj, r.stderr


def test_track_kernel_sums_on_the_fp64_tensor_core(tmp_path):
    obj, _ = _compile(tmp_path)
    r = subprocess.run([CUOBJDUMP, "-sass", "-fun", KERNEL, str(obj)], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr[-3000:]
    dmma = [ln for ln in r.stdout.splitlines() if re.search(r"\bDMMA\.8x8x4\b", ln)]
    # SO(3), ICP and photometric rows, 8 MMAs per 32 pixels each (the phases with two pixels in flight per thread have two tiles)
    assert len(dmma) >= 3 * 8, f"{len(dmma)} DMMA.8x8x4 in k_track_persistent"


def test_track_kernel_spills_stay_small(tmp_path):
    _, log = _compile(tmp_path)
    m = re.search(r"Function properties for " + re.escape(KERNEL) + r"\s*\n\s*\d+ bytes stack frame, (\d+) bytes spill stores, (\d+) bytes spill loads", log)
    assert m, log[-3000:]
    stores, loads = int(m.group(1)), int(m.group(2))
    assert stores <= MAX_SPILL_BYTES and loads <= 3 * MAX_SPILL_BYTES, f"k_track_persistent spills {stores} B stores / {loads} B loads"
