"""Pinned values of the seeded Mask R-CNN handles (mf_backbone, mf_rpn, mf_detector) and the NULL-skip read-backs the header promises.

The digests were recorded on an H100 before the three handles' layer tables, seeded generators and weight stores were merged into one
(mf_weights.cu): every seeded table and bias that *_get_weights returns and the backbone's and the detector's layer tables.  What
Detector.execute returns on one synthetic frame was recorded on an H100 once the input mould followed R-MOLD (DESIGN section 4).  The seeded
tables do not depend on the input size, so S = 256 keeps the test small."""
from __future__ import annotations

import ctypes as C
import hashlib

import numpy as np
import pytest

pytestmark = pytest.mark.gpu
S = 256
W0, H0 = 640, 480

WEIGHTS = {
    ("backbone", 1): "409dc0353d110c52399c9a77fb9371caca4df428cd32d4367ad0af9552bd1b73",
    ("backbone", 7): "8927f1f7d0a55dbfc9e99fd57b7d9c7f42412df0850393570b0cd0aa5836b2e4",
    ("rpn", 1): "03da21dfd3e43684c2af4c3e28e4a50ed432fd33ed33349664d9a0eb28b6b16f",
    ("rpn", 11): "98d8e2e6966cb4d27b33daf235635c1846fd3d20857c241802cbdf0ba81ce676",
    ("detector", 1): "aaa11d69b6e6f514aad4c7bbf91efd3bfe30f46fc5b53540218e8f56c0da7d62",
    ("detector", 13): "7b4d06508ef9d3a0bf6ace8eab9c491c199c3a2fc4d400621aed4c22ecb21aef",
}
LAYERS = {
    "backbone": "7cd5f774dcceb542ec92ce0ae0fb8fa3ff6fca1a2ba28c400ce84a48eded8030",
    "detector": "7406a699e68f54219911d9d3b8c069e2cfaec52ab6e279382fe973c0caf23998",
}
# re-recorded on an H100 when the mould took rule R-MOLD (DESIGN section 4): the network input changed, the tables above did not
EXECUTE = {
    "detections": "484b193209b48f7285aa028b98a25f931e8f955530f5d7d4b0743be53940a99f",
    "masks": "b6b51d73fcd9636a25c3b89f8b493d7f02dfebc6433cb9ebee8aa170eb9ccf89",
    "id_image": "cae983444315591034b79ab214e1f2d464bf62c9aeff3d033eae2917f0d7de2e",
}


def _sha(*arrays) -> str:
    h = hashlib.sha256()
    for a in arrays:
        h.update(np.ascontiguousarray(a).tobytes())
    return h.hexdigest()


def _p(a):
    return a.ctypes.data_as(C.c_void_p)


def _backbone_tables(bb):
    L, out = bb.L, []
    for cin, cout, k, stride, pad, kpad in bb.layers():
        w = np.zeros((cout, kpad), np.float32); b = np.zeros(cout, np.float32)
        assert L.mf_backbone_get_weights(bb.h, len(out) // 2, _p(w), _p(b)) == 0
        out += [w, b]
    return out


def _detector_tables(det):
    return [a for i in range(len(det.layers())) for a in det.weights(i)]


def _nets(bs, rs, ds, stream=None):
    import maskfusion_b200 as mfb
    bb = mfb.Backbone(S, seed=bs, stream=stream)
    rpn = mfb.RegionProposals(bb, seed=rs)
    det = mfb.Detector(rpn, seed=ds)
    return bb, rpn, det


def _close(*hs):
    for h in reversed(hs):
        h.close()


def weight_digests():
    out = {}
    for (bs, rs, ds) in ((1, 1, 1), (7, 11, 13)):
        hs = _nets(bs, rs, ds)
        bb, rpn, det = hs
        out[("backbone", bs)] = _sha(*_backbone_tables(bb))
        out[("rpn", rs)] = _sha(*rpn.weights())
        out[("detector", ds)] = _sha(*_detector_tables(det))
        _close(*hs)
    return out


def layer_digests():
    hs = _nets(1, 1, 1)
    out = {"backbone": _sha(np.array(hs[0].layers(), np.int32)), "detector": _sha(np.array(hs[2].layers(), np.int32))}
    _close(*hs)
    return out


def _executed():
    """the handles at seeds 7, 11, 13 after Detector.execute on the pinned frame -> (backbone, rpn, detector, execute's result)"""
    import torch
    from maskfusion_b200.synth import SynthScene
    rgb, *_ = SynthScene(W0, H0, n_objects=2, seed=5).render(0)
    bb, rpn, det = _nets(7, 11, 13, stream=torch.cuda.current_stream().cuda_stream)
    return bb, rpn, det, det.execute(rgb)


def execute_digests():
    bb, rpn, det, (img, cls, rois) = _executed()
    hs = (bb, rpn, det)
    n, dets = det.detections()
    masks = det.masks()
    _close(*hs)
    assert n > 0 and len(cls) > 0, "the pinned frame must produce detections"
    return {"detections": _sha(np.int32(n), dets), "masks": _sha(masks),
            "id_image": _sha(img, np.array(cls, np.int32), np.array(rois, np.int32).reshape(-1, 4))}


def test_seeded_weight_tables_are_pinned():
    assert weight_digests() == WEIGHTS


def test_layer_tables_are_pinned():
    assert layer_digests() == LAYERS


def test_execute_on_the_r_mold_input_is_pinned():
    assert execute_digests() == EXECUTE


def test_rpn_head_outputs_skip_a_null_destination():
    hs = _executed()
    rpn, L = hs[1], hs[1].L
    lg, dl = rpn.headOutputs()
    lg1 = np.zeros_like(lg); dl1 = np.zeros_like(dl)
    assert L.mf_rpn_get_head_outputs(rpn.h, _p(lg1), None) == 0, L.mf_cnn_last_error()
    assert L.mf_rpn_get_head_outputs(rpn.h, None, _p(dl1)) == 0, L.mf_cnn_last_error()
    _close(*hs[:3])
    np.testing.assert_array_equal(lg1, lg)
    np.testing.assert_array_equal(dl1, dl)


def test_detector_mask_logits_skip_a_null_destination():
    hs = _executed()
    det = hs[2]
    want = det.maskLayer(6)
    assert det.L.mf_detector_get_mask_layer(det.h, 6, None) == 0, det.L.mf_cnn_last_error()
    got = det.maskLayer(6)
    _close(*hs[:3])
    np.testing.assert_array_equal(got, want)
