"""Pretrained Mask R-CNN weights on the GPU (mf_backbone_load_weights, mf_rpn_load_weights, mf_detector_load_weights).

The weight file holds seeded stand-in arrays in matterport's Keras names and layouts (tests/mrcnn_weights_ref.py).  Checked:
  - the device tables after loading equal the numpy R-FOLD + relayout bit for bit, padding included;
  - the network on the loaded weights computes matterport's graph: a torch fp32 restatement built directly from the Keras-layout,
    UNFOLDED arrays (F.conv2d on kernel.permute(3, 2, 0, 1), F.batch_norm in eval mode with eps 1e-3, TF "same" max-pool, nearest x2 top-down,
    F.conv_transpose2d) agrees with the backbone end to end and with every RPN and head GEMM stage on the GPU's own inputs.  The loaded
    weights are bf16 and the restatement's fp32, so every stage is held to the bf16 tolerances of tests/test_gpu_cnn.py / test_gpu_heads.py
    (2^-7 of the largest output; the backbone chain: mean relative error < 6 %);
  - a refused file leaves every table as it was; the frame path with a loaded detector computes what the same frames with its recorded
    masks compute; loading twice gives the same outputs; seeded handles created afterwards are unchanged."""
from __future__ import annotations

import contextlib
import ctypes as C
import importlib.util
import os
import re

import numpy as np
import pytest

from tests import mrcnn_weights_ref as ref

pytestmark = pytest.mark.gpu
W0, H0 = 640, 480
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
TOL = 2.0 ** -7


def _converter():
    spec = importlib.util.spec_from_file_location("convert_mrcnn_h5", os.path.join(ROOT, "scripts", "convert_mrcnn_h5.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


conv = _converter()


@contextlib.contextmanager
def _no_tf32():
    import torch
    saved = torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32
    torch.backends.cudnn.allow_tf32 = False
    torch.backends.cuda.matmul.allow_tf32 = False
    try:
        yield
    finally:
        torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32 = saved


def _frame():
    from maskfusion_b200.synth import SynthScene
    rgb, *_ = SynthScene(W0, H0, n_objects=2, seed=5).render(0)
    return rgb


@pytest.fixture(scope="module")
def weights(tmp_path_factory):
    t = ref.make_weights(21)
    path = str(tmp_path_factory.mktemp("mrcnn") / "mrcnn_stand_in.safetensors")
    conv.write_safetensors(path, t)
    return t, path


@pytest.fixture(scope="module")
def nets(weights):
    """S -> (Backbone, RegionProposals, Detector) with the file's weights after one forward on the moulded synthetic 640x480 frame"""
    import torch
    import maskfusion_b200 as mfb
    made = {}

    def get(S):
        if S not in made:
            bb, rpn, det = mfb.load_mask_rcnn(weights[1], S, stream=torch.cuda.current_stream().cuda_stream)
            rgb = _frame()
            rgba = torch.from_numpy(np.concatenate([rgb, np.full(rgb.shape[:2] + (1,), 255, np.uint8)], axis=2)).cuda()
            L = mfb.load_library()
            assert L.mf_backbone_mold(C.c_void_p(bb.h), C.c_void_p(rgba.data_ptr()), W0, H0) == 0
            bb.forward(L.mf_backbone_input_buffer(bb.h))
            rpn.forward()
            det.forward(W0, H0)
            torch.cuda.synchronize()
            made[S] = (bb, rpn, det)
        return made[S]

    yield get
    for bb, rpn, det in made.values():
        det.close(); rpn.close(); bb.close()


def _backbone_table(bb, i):
    cin, cout, k, stride, pad, kpad = bb.layers()[i]
    w = np.zeros((cout, kpad), np.float32); b = np.zeros(cout, np.float32)
    assert bb.L.mf_backbone_get_weights(bb.h, i, w.ctypes.data_as(C.c_void_p), b.ctypes.data_as(C.c_void_p)) == 0
    return w, b


def _same_bits(a, b, what):
    assert a.shape == b.shape, (what, a.shape, b.shape)
    assert np.array_equal(np.ascontiguousarray(a).view(np.uint32), np.ascontiguousarray(b).view(np.uint32)), what


def _snapshot(bb, rpn, det):
    return ([_backbone_table(bb, i) for i in range(len(bb.layers()))], rpn.weights(), [det.weights(i) for i in range(len(det.layers()))])


def _same_snapshot(a, b):
    for (wa, ba), (wb, bb_) in zip(a[0], b[0]):
        _same_bits(wa, wb, "backbone"); _same_bits(ba, bb_, "backbone bias")
    for x, y in zip(a[1], b[1]):
        _same_bits(x, y, "rpn")
    for (wa, ba), (wb, bb_) in zip(a[2], b[2]):
        _same_bits(wa, wb, "detector"); _same_bits(ba, bb_, "detector bias")


def test_tables_equal_the_numpy_fold(nets, weights):
    t, _ = weights
    bb, rpn, det = nets(256)
    tabs = ref.handle_tables()
    assert len(bb.layers()) == len(tabs["backbone"]) == 112
    for i, (name, _, rows, K) in enumerate(tabs["backbone"]):
        w, b = _backbone_table(bb, i)
        W, B = ref.table(t, name)
        _same_bits(w, W, name); _same_bits(b, B, name)
    cw, cb, hw, hb = rpn.weights()
    W, B = ref.table(t, "rpn_conv_shared")
    _same_bits(cw.reshape(512, -1), W, "rpn_conv_shared"); _same_bits(cb, B, "rpn_conv_shared")
    W, B = ref.table(t, "rpn_class_raw+rpn_bbox_pred")
    _same_bits(hw, W[:18], "rpn head"); _same_bits(hb, B[:18], "rpn head")
    assert not W[18:].any() and not B[18:].any()
    for i, (name, _, rows, K) in enumerate(tabs["detector"]):
        w, b = det.weights(i)
        W, B = ref.table(t, name)
        _same_bits(w, W, name); _same_bits(b, B, name)


# ---- the torch restatement of matterport's graph on the Keras-layout, unfolded arrays -------------------------------------------------
class Keras:
    def __init__(self, t):
        import torch
        self.t, self.torch = t, torch
        self.bn = {n: bn for layers in ref.ALL_LAYERS.values() for n, bn, _ in layers}

    def a(self, name):
        return self.torch.from_numpy(self.t[name]).cuda()

    def conv(self, x, name, stride=1, padding=0, relu=True, residual=None, bf16=True):
        """Conv2D (+ BatchNorm in inference mode) (+ residual) (+ ReLU) on NCHW x; bf16 storage of the result as on the GPU"""
        import torch.nn.functional as F
        y = F.conv2d(x.float(), self.a(name + "/kernel").permute(3, 2, 0, 1), self.a(name + "/bias"), stride=stride, padding=padding)
        bn = self.bn[name]
        if bn:
            y = F.batch_norm(y, self.a(bn + "/moving_mean"), self.a(bn + "/moving_variance"), self.a(bn + "/gamma"), self.a(bn + "/beta"),
                             training=False, eps=ref.EPS)
        if residual is not None:
            y = y + residual.float()
        if relu:
            y = self.torch.relu(y)
        return y.to(self.torch.bfloat16) if bf16 else y

    def dense(self, x, name):
        return x.float() @ self.a(name + "/kernel") + self.a(name + "/bias")


def _moulded_input(torch, bb):
    """the GPU's moulded network input [S, S, 3] bf16, read from the backbone's input buffer"""
    S = bb.S

    class Dev:
        __cuda_array_interface__ = {"shape": (S, S, 3), "typestr": "<i2", "data": (bb.L.mf_backbone_input_buffer(bb.h), False), "version": 2}
    return torch.as_tensor(Dev(), device="cuda").clone().view(torch.bfloat16)


def _rel_check(got, want, what, tol=TOL):
    err, scale = float((got - want).abs().max()), float(want.abs().max())
    assert scale > 1e-2, (what, "degenerate output")
    assert err <= tol * max(scale, 1.0), (what, err, scale)


@pytest.mark.parametrize("S", [256, 1024])
def test_backbone_computes_matterport_graph(nets, weights, S):
    """resnet_graph(resnet101, stage5=True) + FPN from the moulded input, compared at C2..C5 and P2..P6 as tests/test_gpu_cnn.py does"""
    import torch
    import torch.nn.functional as F
    bb, rpn, det = nets(S)
    k = Keras(weights[0])
    with _no_tf32():
        x = _moulded_input(torch, bb).permute(2, 0, 1)[None]
        x = k.conv(x, "conv1", stride=2, padding=3)
        x = F.max_pool2d(F.pad(x.float(), (0, 1, 0, 1), value=float("-inf")), 3, 2).to(torch.bfloat16)      # TF "same": pad after only
        Cs = []
        for st, nb in ((2, 3), (3, 4), (4, 23), (5, 3)):
            for blk in range(nb):
                n = f"res{st}{chr(ord('a') + blk)}_branch"
                s = 2 if blk == 0 and st > 2 else 1
                y = k.conv(k.conv(x, n + "2a", stride=s), n + "2b", padding=1)
                sc = k.conv(x, n + "1", stride=s, relu=False) if blk == 0 else x
                x = k.conv(y, n + "2c", residual=sc)
            Cs.append(x)
        top = k.conv(Cs[3], "fpn_c5p5", relu=False)
        P = [None] * 5
        P[3] = k.conv(top, "fpn_p5", padding=1, relu=False)
        for i in (2, 1, 0):
            lat = k.conv(Cs[i], f"fpn_c{i + 2}p{i + 2}", relu=False)
            top = (lat.float() + F.interpolate(top.float(), scale_factor=2, mode="nearest")).to(torch.bfloat16)
            P[i] = k.conv(top, f"fpn_p{i + 2}", padding=1, relu=False)
        P[4] = P[3][:, :, ::2, ::2]                                            # P6: MaxPooling2D(1, strides=2)
    report = {}
    for lvl in range(9):
        got = torch.from_numpy(bb.download(lvl)).cuda()
        want = (Cs[lvl] if lvl < 4 else P[lvl - 4])[0].permute(1, 2, 0).float()
        assert not torch.isnan(got).any(), lvl
        report[lvl] = ((got - want).abs().mean().item() / (want.abs().mean().item() + 1e-6), want.abs().mean().item())
    print("mean relative error, mean |activation| per level C2..C5 P2..P6:", report)
    for lvl, (rel, mag) in report.items():
        assert mag > 1e-3, (lvl, "degenerate activations", report)
        assert rel < 0.06, report


@pytest.mark.parametrize("S", [256, 1024])
def test_rpn_computes_matterport_graph(nets, weights, S):
    """rpn_graph on the GPU's P2..P6: shared 3x3 conv + ReLU, then rpn_class_raw (channel a*2 + c) and rpn_bbox_pred (a*4 + k)"""
    import torch
    bb, rpn, det = nets(S)
    k = Keras(weights[0])
    lgs, dls = [], []
    with _no_tf32():
        for lvl in range(5):
            p = torch.from_numpy(bb.download(4 + lvl)).cuda().permute(2, 0, 1)[None]
            want = k.conv(p, "rpn_conv_shared", padding=1, bf16=False)[0].permute(1, 2, 0)
            got = torch.from_numpy(rpn.convOutput(lvl)).cuda()
            _rel_check(got, want, ("rpn conv", lvl))
            g = got.permute(2, 0, 1)[None]
            lgs.append(k.conv(g, "rpn_class_raw", relu=False, bf16=False)[0].permute(1, 2, 0).reshape(-1, 6))
            dls.append(k.conv(g, "rpn_bbox_pred", relu=False, bf16=False)[0].permute(1, 2, 0).reshape(-1, 12))
    lg, dl = rpn.headOutputs()
    _rel_check(torch.from_numpy(lg.reshape(-1, 6)).cuda(), torch.cat(lgs), "rpn logits")
    _rel_check(torch.from_numpy(dl.reshape(-1, 12)).cuda(), torch.cat(dls), "rpn deltas")


@pytest.mark.parametrize("S", [256, 1024])
def test_heads_compute_matterport_graph(nets, weights, S):
    """fpn_classifier_graph and build_fpn_mask_graph stage by stage on the GPU's own inputs: FC1 (7x7 valid conv + BN + ReLU), FC2, class
    logits and box deltas (Dense), the four mask convs (3x3 same + BN + ReLU), the transposed conv and the mask logits"""
    import torch
    import torch.nn.functional as F
    bb, rpn, det = nets(S)
    k = Keras(weights[0])
    fc1, fc2 = det.fcOutputs()
    with _no_tf32():
        x = torch.from_numpy(rpn.pooled()).cuda().permute(0, 3, 1, 2)
        _rel_check(torch.from_numpy(fc1).cuda(), k.conv(x, "mrcnn_class_conv1", bf16=False).reshape(1000, 1024), "FC1")
        x = torch.from_numpy(fc1).cuda().reshape(1000, 1024, 1, 1)
        _rel_check(torch.from_numpy(fc2).cuda(), k.conv(x, "mrcnn_class_conv2", bf16=False).reshape(1000, 1024), "FC2")
        x = torch.from_numpy(fc2).cuda()
        lg, dl = det.headOutputs()
        _rel_check(torch.from_numpy(lg).cuda(), k.dense(x, "mrcnn_class_logits"), "class logits")
        _rel_check(torch.from_numpy(dl).cuda(), k.dense(x, "mrcnn_bbox_fc").reshape(1000, 81, 4), "box deltas")
        prev = det.maskLayer(0)
        for i in range(4):
            x = torch.from_numpy(prev).cuda().permute(0, 3, 1, 2)
            want = k.conv(x, f"mrcnn_mask_conv{i + 1}", padding=1, bf16=False).permute(0, 2, 3, 1)
            prev = det.maskLayer(1 + i)
            _rel_check(torch.from_numpy(prev).cuda(), want, ("mask conv", i))
        x = torch.from_numpy(prev).cuda().permute(0, 3, 1, 2)
        want = torch.relu(F.conv_transpose2d(x, k.a("mrcnn_mask_deconv/kernel").permute(3, 2, 0, 1), k.a("mrcnn_mask_deconv/bias"), stride=2))
        dec = det.maskLayer(5)                                                  # [d][y][x][dy][dx][c]
        _rel_check(torch.from_numpy(dec).cuda().permute(0, 5, 1, 3, 2, 4).reshape(100, 256, 28, 28), want, "transposed conv")
        x = torch.from_numpy(dec).cuda().permute(0, 5, 1, 3, 2, 4).reshape(100, 256, 28, 28)
        want = k.conv(x, "mrcnn_mask", relu=False, bf16=False)                 # [d][81][28][28]
        got = torch.from_numpy(det.maskLayer(6)).cuda().permute(0, 5, 1, 3, 2, 4).reshape(100, 81, 28, 28)
        _rel_check(got, want, "mask logits")
    n, dets = det.detections()
    print(f"S={S}: {n} detections, classes {sorted(set(dets[:n, 4].astype(int).tolist()))}")


# ---- all or nothing ---------------------------------------------------------------------------------------------------------------------
VICTIMS = {"backbone": "fpn_p5/kernel", "rpn": "rpn_bbox_pred/bias", "detector": "mrcnn_mask/kernel"}    # read last by each loader


@pytest.mark.parametrize("kind", ["missing", "shape", "f16"])
def test_refused_file_leaves_the_tables(weights, tmp_path, kind):
    import torch
    import maskfusion_b200 as mfb
    t, _ = weights
    st = torch.cuda.Stream()
    bb = mfb.Backbone(256, seed=7, stream=st.cuda_stream)
    rpn = mfb.RegionProposals(bb, seed=11)
    det = mfb.Detector(rpn, seed=13)
    try:
        before = _snapshot(bb, rpn, det)
        for (part, victim), h in zip(VICTIMS.items(), (bb, rpn, det)):
            names = {f"{n}/{p}" for n, bn, _ in ref.ALL_LAYERS[part] for p in ("kernel", "bias")}
            names |= {f"{bn}/{p}" for n, bn, _ in ref.ALL_LAYERS[part] if bn for p in ("gamma", "beta", "moving_mean", "moving_variance")}
            sub = {n: t[n] for n in names}
            if kind == "missing":
                del sub[victim]
            elif kind == "shape":
                sub[victim] = sub[victim][..., :-1].copy()
            else:
                sub[victim] = sub[victim].astype(np.float16)
            path = str(tmp_path / f"{part}.safetensors")
            conv.write_safetensors(path, sub)
            with pytest.raises(mfb.MFError, match=re.escape(f"tensor '{victim}'")) as e:
                h.loadWeights(path)
            assert path in str(e.value)
            os.remove(path)
        _same_snapshot(_snapshot(bb, rpn, det), before)
    finally:
        det.close(); rpn.close(); bb.close()


# ---- frame path, reloading, no leaked state ------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def frames():
    from maskfusion_b200.synth import SynthScene
    from tests.test_gpu_detect_frame import H, N_FRAMES, W
    sc = SynthScene(W, H, n_objects=3, seed=0, layout="table")
    out = []
    for t in range(N_FRAMES):
        rgb, depth, mask, *_ = sc.render(t)
        out.append((np.ascontiguousarray(rgb), np.ascontiguousarray(depth), np.ascontiguousarray(mask)))
    return out


def test_frame_path_with_loaded_weights(weights, frames):
    """tests/test_gpu_detect_frame.py's pair at S = 256, every_k = 1, on loaded weights: a context with the detector attached and a context
    fed its recorded frameMasks() agree bit for bit in poses, segmentation, surfel counts and stores"""
    import torch
    import maskfusion_b200 as mfb
    from tests.test_gpu_detect_frame import _check_handoff, _run_pair
    st = torch.cuda.Stream()
    bb, rpn, det = mfb.load_mask_rcnn(weights[1], 256, stream=st.cuda_stream)
    try:
        det.set_export()
        recs = _run_pair(det, frames, None, 1, False)
        _check_handoff(recs)
        ran = [len(r["ids"]) - 1 for r in recs if r["ran"]]
        print("exported detections per detector frame:", ran, "models at the end:", recs[-1]["models"])
        assert len(ran) == len(frames) - 1 and max(ran) >= 1, ran
    finally:
        det.close(); rpn.close(); bb.close()


def test_reload_and_fresh_seeded_handles(weights):
    """loading the same file again gives the same outputs bit for bit; seeded handles created after loads equal those created before"""
    import torch
    import maskfusion_b200 as mfb
    st = torch.cuda.Stream()

    def seeded():
        bb = mfb.Backbone(256, seed=7, stream=st.cuda_stream)
        rpn = mfb.RegionProposals(bb, seed=11)
        return bb, rpn, mfb.Detector(rpn, seed=13)

    def close(hs):
        for h in reversed(hs):
            h.close()

    def outputs(det):
        img, cls, rois = det.execute(_frame())
        n, dets = det.detections()
        return img, cls, rois, n, dets, det.masks(), det.headOutputs()[0]

    hs = seeded()
    before = _snapshot(*hs)
    close(hs)
    hs = mfb.load_mask_rcnn(weights[1], 256, stream=st.cuda_stream)
    try:
        a = outputs(hs[2])
        for h in hs:
            h.loadWeights(weights[1])
        b = outputs(hs[2])
    finally:
        close(hs)
    assert np.array_equal(a[0], b[0]) and a[1] == b[1] and a[2] == b[2] and a[3] == b[3]
    for x, y in zip(a[4:], b[4:]):
        _same_bits(x, y, "reload")
    hs = seeded()
    try:
        _same_snapshot(_snapshot(*hs), before)
    finally:
        close(hs)


def test_converted_coco_file_if_present():
    """MFB200_MRCNN_WEIGHTS = a file converted from matterport's mask_rcnn_coco.h5 (scripts/convert_mrcnn_h5.py): it passes validation at
    S = 1024 and the detector runs on a synthetic frame"""
    path = os.environ.get("MFB200_MRCNN_WEIGHTS")
    if not path:
        pytest.skip("MFB200_MRCNN_WEIGHTS is not set")
    import torch
    import maskfusion_b200 as mfb
    bb, rpn, det = mfb.load_mask_rcnn(path, 1024, stream=torch.cuda.current_stream().cuda_stream)
    try:
        img, cls, rois = det.execute(_frame())
        assert img.shape == (H0, W0) and len(cls) == len(rois)
        print("COCO weights on the synthetic frame: classes", cls)
    finally:
        det.close(); rpn.close(); bb.close()
