"""Compile-time guard of the persistent tracker's local-memory use (no GPU needed: nvcc cross-compiles for sm_90a).

k_track_persistent runs up to 48 grid-wide fp64 reductions per frame, each a link of a dependent chain.  When the halving shuffle tree's
value array stopped being unrolled, it was indexed at run time and lived in local memory: 480 bytes of stack per thread, the
reductions four times slower, and nothing but the frame rate showed it.  These tests read what the compiler made of the kernel."""
import os
import re
import shutil
import subprocess

import pytest

from maskfusion_b200 import build as B

KERNEL = "_ZN3mfb18k_track_persistentEPKNS_8TrackJobENS_11TrackParamsE"
SRC = os.path.join(B.CSRC, "mf_track.cu")
# register spills only (the kernel is capped at 128 registers by __launch_bounds__(512, 1)); 480 bytes when the reduction tree's values
# sat in local memory
MAX_STACK_BYTES = 256

pytestmark = pytest.mark.skipif(not shutil.which(B.NVCC) and not os.path.exists(B.NVCC), reason="nvcc not available")


def _nvcc(tmp_path, *args):
    cmd = [B.NVCC] + B.ARCH + B.COMMON + B.SOURCES["mf_track.cu"] + ["-I", B.CSRC] + list(args) + [SRC]
    r = subprocess.run(cmd, capture_output=True, text=True, cwd=tmp_path)
    assert r.returncode == 0, r.stderr[-3000:]
    return r


def test_track_kernel_has_no_local_arrays(tmp_path):
    """every per-thread array of the kernel is indexed with constants (held in registers): its PTX has no local loads or stores"""
    ptx = tmp_path / "mf_track.ptx"
    _nvcc(tmp_path, "-ptx", "-o", str(ptx))
    text = ptx.read_text()
    start = text.index(".entry " + KERNEL)
    body = text[start:text.index("\n}\n", start)]
    local = [ln.strip() for ln in body.splitlines() if re.search(r"\b(ld|st)\.local\b", ln)]
    assert not local, f"{len(local)} local-memory accesses in the PTX of k_track_persistent, e.g. {local[:4]}"


def test_track_kernel_stack_bound(tmp_path):
    r = _nvcc(tmp_path, "-c", "-o", str(tmp_path / "mf_track.o"), "-Xptxas", "-v")
    m = re.search(r"Function properties for " + re.escape(KERNEL) + r"\s*\n\s*(\d+) bytes stack frame", r.stderr)
    assert m, r.stderr[-3000:]
    assert int(m.group(1)) <= MAX_STACK_BYTES, f"k_track_persistent: {m.group(1)} bytes stack frame (bound {MAX_STACK_BYTES})"
