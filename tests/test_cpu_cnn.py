"""The geometry rule of the implicit 3x3 convolution (csrc/mf_cnn.cu, cnn_conv_implicit) seen through mf_conv3x3_bf16: a shape whose
128-pixel TMA box does not tile the image would leave the GEMM's full barrier waiting for bytes that never arrive, so the entry point has to
refuse it before any driver call.  The calls run in a subprocess that sees no CUDA device and pass null pointers: a refusal that regressed
could not reach a GPU."""
from __future__ import annotations

import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

# (H, W, Cin, Cout): W < 128 that does not divide 128, W below the 8-pixel box, empty and negative sides, Cin off 64, W > 128 off 128
REFUSED = [(48, 48, 64, 64), (80, 80, 64, 64), (96, 96, 64, 64), (24, 24, 64, 64), (16, 80, 256, 128), (96, 24, 64, 64),
           (64, 4, 64, 64), (32, 0, 64, 64), (0, 32, 64, 64), (0, 0, 64, 64), (-8, 16, 64, 64), (16, -16, 64, 64), (-1, -1, 64, 64),
           (16, 16, 96, 64), (16, 16, 32, 64), (16, 16, 0, 64), (16, 16, -64, 64), (2, 200, 64, 64), (1, 192, 64, 64), (1, 1000, 64, 64),
           (3, 16, 64, 64), (1, 64, 64, 64)]

_CHILD = r"""
import ctypes as C, json, sys
import maskfusion_b200 as mfb
L = mfb.load_library()
out = []
for H, W, Cin, Cout in json.loads(sys.argv[1]):
    rc = L.mf_conv3x3_bf16(None, None, None, None, None, H, W, Cin, Cout, 1, None)
    out.append([rc, L.mf_cnn_last_error().decode()])
print(json.dumps(out))
"""


def test_conv3x3_refuses_untileable_geometry_without_a_device(product_lib):
    env = dict(os.environ, CUDA_VISIBLE_DEVICES="")
    r = subprocess.run([sys.executable, "-c", _CHILD, json.dumps(REFUSED)], capture_output=True, text=True, env=env, cwd=ROOT, timeout=300)
    assert r.returncode == 0, r.stderr
    got = json.loads(r.stdout.strip().splitlines()[-1])
    for shape, (rc, msg) in zip(REFUSED, got):
        assert (rc, msg) == (-2, "conv3x3: unsupported geometry"), shape
