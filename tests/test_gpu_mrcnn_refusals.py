"""Refusals of the Mask R-CNN entry points that need a live handle, and the backbone on a second device.

Each refusal keeps its return code and its text, and leaves the handle as it was: after the table the same handles still give the digests
that tests/test_gpu_mrcnn_tables.py pins.  The GEMM launcher sets the wgmma kernel's shared-memory attribute per device, so a backbone on a
second GPU of the same process runs and computes what the first one does."""
from __future__ import annotations

import ctypes as C
import json
import os
import subprocess
import sys

import numpy as np
import pytest

from tests import test_gpu_mrcnn_tables as tables

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_refusals_with_live_handles_keep_code_text_and_state():
    import torch
    from maskfusion_b200.synth import SynthScene
    bb, rpn, det = tables._nets(7, 11, 13, stream=torch.cuda.current_stream().cuda_stream)
    L, i6, ids = bb.L, (C.c_int * 6)(), (C.c_int32 * 129)()
    A = L.mf_rpn_num_anchors(rpn.h)
    table = [
        (lambda: L.mf_backbone_layer(bb.h, 999, i6), "backbone: bad layer index"),
        (lambda: L.mf_backbone_get_weights(bb.h, 999, None, None), "backbone: bad layer index"),
        (lambda: L.mf_detector_layer(det.h, 9, i6), "detector: bad layer index"),
        (lambda: L.mf_detector_get_weights(det.h, 9, None, None), "detector: bad layer index"),
        (lambda: L.mf_backbone_mold(bb.h, None, 0, 480), "mold: the image needs W > 0 and H > 0"),
        (lambda: L.mf_backbone_download(bb.h, 9, None), "backbone: no handle or level outside 0..8"),
        (lambda: L.mf_rpn_propose(rpn.h, None, None, None, 0), f"rpn_propose: n_anchors = 0 outside [1, {A}]"),
        (lambda: L.mf_rpn_download_conv(rpn.h, 5, None), "rpn: level must be 0..4 (P2..P6)"),
        (lambda: L.mf_roi_align_bf16(bb.h, None, 1, 1, None), "roi_align: need n >= 0 and 2 <= pool <= 64"),
        (lambda: L.mf_detector_refine(det.h, None, None, None, 0), "detector_refine: n = 0 outside [1, 1000]"),
        (lambda: L.mf_detector_refine(det.h, None, None, None, 1001), "detector_refine: n = 1001 outside [1, 1000]"),
        (lambda: L.mf_detector_forward(det.h, 0, 10), "detector: image size 0x10 outside [1, 16384]"),
        (lambda: L.mf_detector_forward(det.h, 16385, 1), "detector: image size 16385x1 outside [1, 16384]"),
        (lambda: L.mf_detector_set_export(det.h, 0.5, ids, 129, None, 0), "detector_set_export: lists of 0..128 entries"),
        (lambda: L.mf_detector_get_mask_layer(det.h, 7, None), "detector: mask layer must be 0..6"),
    ]
    got = [(call(), L.mf_last_error().decode()) for call, _ in table]
    assert got == [(-1, text) for _, text in table]
    rgb, *_ = SynthScene(tables.W0, tables.H0, n_objects=2, seed=5).render(0)
    img, cls, rois = det.execute(rgb)
    n, dets = det.detections()
    digests = {"detections": tables._sha(np.int32(n), dets), "masks": tables._sha(det.masks()),
               "id_image": tables._sha(img, np.array(cls, np.int32), np.array(rois, np.int32).reshape(-1, 4))}
    weights = {("backbone", 7): tables._sha(*tables._backbone_tables(bb)), ("rpn", 11): tables._sha(*rpn.weights()),
               ("detector", 13): tables._sha(*tables._detector_tables(det))}
    tables._close(bb, rpn, det)
    assert digests == tables.EXECUTE
    assert weights == {k: tables.WEIGHTS[k] for k in weights}


_TWO_DEVICES = r"""
import ctypes as C, hashlib, json
import numpy as np, torch
import maskfusion_b200 as mfb
S, out = 256, []
for dev in (0, 1):
    torch.cuda.set_device(dev)
    g = torch.Generator(device="cpu").manual_seed(3)
    x = (torch.rand(S, S, 3, generator=g) * 200 - 100).to(torch.bfloat16).cuda(dev)
    bb = mfb.Backbone(S, seed=3, stream=torch.cuda.current_stream(dev).cuda_stream)
    rc = bb.L.mf_backbone_forward(bb.h, C.c_void_p(x.data_ptr()))
    err = bb.L.mf_last_error().decode()
    levels = []
    for lv in range(4, 9):
        _, (h, w, c) = bb.output(lv)
        raw = np.zeros((h, w, c), np.uint16)
        bb.L.mf_backbone_download(bb.h, lv, raw.ctypes.data_as(C.c_void_p))
        levels.append(hashlib.sha256(raw.tobytes()).hexdigest() if rc == 0 else "")
    out.append([rc, err if rc else "", levels])
    bb.close()
print(json.dumps(out))
"""


def test_backbone_runs_on_a_second_device():
    import torch
    if torch.cuda.device_count() < 2:
        pytest.skip("needs two CUDA devices")
    r = subprocess.run([sys.executable, "-c", _TWO_DEVICES], capture_output=True, text=True, cwd=ROOT, timeout=600)
    assert r.returncode == 0, r.stderr
    (rc0, err0, p0), (rc1, err1, p1) = json.loads(r.stdout.strip().splitlines()[-1])
    assert (rc0, err0) == (0, "") and (rc1, err1) == (0, "")
    assert p1 == p0
