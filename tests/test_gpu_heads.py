"""Detection heads on the GPU (csrc/mf_heads.cu): classifier, detection layer, mask head, unmould + id image.

The GEMMs (FC1, FC2, the fp32 class/delta heads, the mask convs, the transposed conv and the mask logits) are checked against PyTorch fp32
with the tolerances of tests/test_gpu_rpn.py.  Everything after the GEMMs is compared bit for bit with the numpy restatement
(tests/heads_ref.py), run on the GPU's own GEMM outputs, proposals and P-level maps."""
from __future__ import annotations

import contextlib
import ctypes as C
import zlib

import numpy as np
import pytest

from tests import heads_ref as ref
from tests import rpn_ref

pytestmark = pytest.mark.gpu
f32 = np.float32
W0, H0 = 640, 480


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
def nets():
    """S -> (Backbone, RegionProposals, Detector) after one forward on the moulded synthetic 640x480 frame of the RPN tests"""
    import torch
    import maskfusion_b200 as mfb
    made = {}

    def get(S):
        if S not in made:
            bb = mfb.Backbone(S, seed=7, stream=torch.cuda.current_stream().cuda_stream)
            rgb = _frame()
            rgba = torch.from_numpy(np.concatenate([rgb, np.full(rgb.shape[:2] + (1,), 255, np.uint8)], axis=2)).cuda()
            L = mfb.load_library()
            assert L.mf_backbone_mold(C.c_void_p(bb.h), C.c_void_p(rgba.data_ptr()), W0, H0) == 0
            bb.forward(L.mf_backbone_input_buffer(bb.h))
            rpn = mfb.RegionProposals(bb, seed=11)
            rpn.forward()
            det = mfb.Detector(rpn, seed=13)
            det.forward(W0, H0)
            torch.cuda.synchronize()
            made[S] = (bb, rpn, det)
        bb, rpn, det = made[S]
        det.set_export()
        return made[S]

    yield get
    for bb, rpn, det in made.values():
        det.close()
        rpn.close()
        bb.close()


def _rel_check(got, want, tol, what):
    err, scale = float((got - want).abs().max()), float(want.abs().max())
    assert scale > 1e-2, (what, "degenerate output")
    assert err <= tol * max(scale, 1.0), (what, err, scale)


def _window(det):
    img, _, _ = det.idImage()
    return ref.window(det.rpn.S, img.shape[1], img.shape[0])


@pytest.mark.parametrize("S", [256, 1024])
def test_fc_layers_match_torch(nets, S):
    """FC1 (7x7 valid conv read as a GEMM on the pooled ROIs, K = 12 544) and FC2 against torch fp32 on the GPU's own inputs"""
    import torch
    bb, rpn, det = nets(S)
    fc1, fc2 = det.fcOutputs()
    X = torch.from_numpy(rpn.pooled().reshape(1000, -1)).cuda()
    with _no_tf32():
        for (w, b), x, got in ((det.weights(0), X, fc1), (det.weights(1), torch.from_numpy(fc1).cuda(), fc2)):
            want = torch.relu(x @ torch.from_numpy(w).cuda().t() + torch.from_numpy(b).cuda()[None])
            _rel_check(torch.from_numpy(got).cuda(), want, 2.0 ** -7, w.shape)


@pytest.mark.parametrize("S", [256, 1024])
def test_class_and_delta_heads_fp32_match_torch(nets, S):
    import torch
    bb, rpn, det = nets(S)
    _, fc2 = det.fcOutputs()
    w, b = det.weights(2)
    with _no_tf32():
        want = torch.from_numpy(fc2).cuda() @ torch.from_numpy(w[:405]).cuda().t() + torch.from_numpy(b[:405]).cuda()[None]
    lg, dl = det.headOutputs()
    got = torch.from_numpy(np.concatenate([lg, dl.reshape(1000, -1)], axis=1)).cuda()
    _rel_check(got, want, 1e-4, "heads")
    assert not w[405:].any() and not b[405:].any()


@pytest.mark.parametrize("S", [256, 1024])
def test_mask_head_layers_match_torch(nets, S):
    """ROI Align at 14 of the detection boxes bit for bit; each 3x3 conv against F.conv2d per ROI on the GPU's previous layer, the transposed
    conv against F.conv_transpose2d, the mask logits against fp32 torch"""
    import torch
    import torch.nn.functional as F
    bb, rpn, det = nets(S)
    n, dets = det.detections()
    pooled_raw = det.maskLayer(0)
    want_pool = rpn_ref.roi_align([bb.download(4 + i) for i in range(4)], dets[:, :4], 14, S)
    assert np.array_equal(rpn_ref.to_bf16_bits(pooled_raw), want_pool)
    prev = pooled_raw
    with _no_tf32():
        for i in range(4):
            w, b = det.weights(3 + i)
            wt = torch.from_numpy(w.reshape(256, 3, 3, 256)).cuda().permute(0, 3, 1, 2)
            x = torch.from_numpy(prev).cuda().permute(0, 3, 1, 2)
            want = torch.relu(F.conv2d(x, wt, torch.from_numpy(b).cuda(), padding=1)).permute(0, 2, 3, 1)
            got = det.maskLayer(1 + i)
            _rel_check(torch.from_numpy(got).cuda(), want, 2.0 ** -7, ("conv", i))
            prev = got
        w, b = det.weights(7)                                           # rows (dy * 2 + dx) * 256 + cout, K = cin
        wt = torch.from_numpy(w.reshape(2, 2, 256, 256)).cuda().permute(3, 2, 0, 1)      # [cin][cout][dy][dx]
        x = torch.from_numpy(prev).cuda().permute(0, 3, 1, 2)
        want = torch.relu(F.conv_transpose2d(x, wt, torch.from_numpy(b[:256]).cuda(), stride=2))       # [d][c][2y+dy][2x+dx]
        dec = det.maskLayer(5)                                          # [d][y][x][dy][dx][c]
        got = torch.from_numpy(dec).cuda().permute(0, 5, 1, 3, 2, 4).reshape(100, 256, 28, 28)
        _rel_check(got, want, 2.0 ** -7, "transposed conv")
        w, b = det.weights(8)
        want = torch.from_numpy(dec.reshape(-1, 256)).cuda() @ torch.from_numpy(w[:81]).cuda().t() + torch.from_numpy(b[:81]).cuda()[None]
        _rel_check(torch.from_numpy(det.maskLayer(6).reshape(-1, 81)).cuda(), want, 1e-4, "mask logits")


def _forward_reference(det, S):
    lg, dl = det.headOutputs()
    _, rois = det.rpn.proposals()
    return ref.detection_layer(rois, lg, dl, ref.window(S, W0, H0))


@pytest.mark.parametrize("S", [256, 1024])
def test_detections_bit_exact(nets, S):
    bb, rpn, det = nets(S)
    n, dets = det.detections()
    rn, rdets, _ = _forward_reference(det, S)
    assert n == rn, (n, rn)
    assert np.array_equal(dets.view(np.uint32), rdets.view(np.uint32)), np.argwhere(dets.view(np.uint32) != rdets.view(np.uint32))[:5]


@pytest.mark.parametrize("S", [256, 1024])
def test_masks_bit_exact(nets, S):
    bb, rpn, det = nets(S)
    _, dets = det.detections()
    want = ref.select_masks(det.maskLayer(6), dets)
    assert np.array_equal(det.masks().view(np.uint32), want.view(np.uint32))


def _exports(dets):
    """(min_score, class_filter, special_assignments): the defaults, and 0.9 with a class filter and a special assignment"""
    classes = sorted({int(c) for c in dets[:, 4] if c > 0})
    c0 = classes[0] if classes else 1
    special = [200 + i for i in range(81)]
    special[c0] = 7                                    # c0 occurs in the list (at index 7): its detections get id special[c0] = 7, and
    special[7] = c0                                    # class 7 (at index c0) gets id c0; the values 200.. are no class ids
    return [(0.55, (), ()), (0.9, tuple(classes[:3]) or (1,), tuple(special))]


@pytest.mark.parametrize("S", [256, 1024])
def test_id_image_bit_exact(nets, S):
    bb, rpn, det = nets(S)
    _, dets = det.detections()
    masks = det.masks()
    for ms, cf, sa in _exports(dets):
        det.set_export(ms, cf, sa)
        det.run(det.ID_IMAGE)
        img, cls, rois = det.idImage()
        rimg, rcls, rrois = ref.id_image(dets, masks, ref.window(S, W0, H0), W0, H0, ms, cf, sa)
        assert img.shape == (H0, W0)
        assert cls == rcls and rois == rrois, (ms, cls, rcls)
        assert np.array_equal(img, rimg), (ms, int((img != rimg).sum()))
    det.set_export()
    det.run(det.ID_IMAGE)


def test_outputs_not_degenerate(nets):
    """the seeded weights give several confident detections of several classes, per-class NMS has work to do, masks split inside their boxes"""
    bb, rpn, det = nets(1024)
    n, dets = det.detections()
    _, _, removed = _forward_reference(det, 1024)
    assert n >= 3 and len(set(dets[:n, 4].tolist())) >= 2, (n, dets[:n, 4])
    assert removed >= 1
    masks = det.masks()
    win = ref.window(1024, W0, H0)
    split = 0
    for d, y1, x1, y2, x2, _, _ in ref.unmold(dets, win, W0, H0):
        inside = ref.resize_mask(masks[d], y2 - y1, x2 - x1) >= 0.5
        split += bool(inside.any() and not inside.all())
    assert split >= 1
    img, cls, _ = det.idImage()
    assert len(set(np.unique(img).tolist()) - {0}) >= 2, np.unique(img)


def _boxes(rng, n, lo=0.0, hi=1.0, smin=0.02, smax=0.3):
    c = rng.uniform(lo, hi, (n, 2)); s = rng.uniform(smin, smax, (n, 2))
    return np.concatenate([c - s / 2, c + s / 2], axis=1).astype(np.float32)


def _grid_boxes(n, side=0.02):
    """n small disjoint boxes on a grid inside the window"""
    k = int(np.ceil(np.sqrt(n)))
    i = np.arange(n)
    y, x = 0.3 + (i // k) * 0.4 / k, 0.05 + (i % k) * 0.9 / k
    return np.stack([y, x, y + side, x + side], 1).astype(np.float32)


def _confident(rng, n, classes, margin=8.0):
    lg = rng.normal(0, 1, (n, 81))
    lg[np.arange(n), classes] += margin + rng.uniform(0, 2, n)
    return lg


def _refine_case(case):
    rng = np.random.default_rng(zlib.crc32(case.encode()))
    n = 1000
    dl = rng.normal(0, 1, (n, 81, 4))
    rois = _boxes(rng, n)
    if case == "score_ties":                  # three logit patterns: equal scores within a class, across classes, and two-way ties in a row
        pat = rng.integers(0, 3, n)
        lg = np.zeros((n, 81))
        cls = rng.integers(1, 81, n)
        lg[np.arange(n), cls] = 9.0
        lg[pat == 1, :] = 0.0
        lg[pat == 1, 5] = 9.0                 # same score as pattern 0, class 5
        lg[pat == 2, 3] = 9.0; lg[pat == 2, 4] = 9.0      # tie inside the row: class 3 (lowest index) with probability < 0.7 -> dropped
        rois = _boxes(rng, n, smin=0.05, smax=0.2)
    elif case == "nan_logits":
        lg = _confident(rng, n, rng.integers(1, 81, n))
        lg[rng.choice(n, 200, replace=False), rng.integers(0, 81, 200)] = np.nan
        lg[:10, 0] = np.nan                   # NaN first: the max starts at NaN
    elif case == "all_background":
        lg = _confident(rng, n, np.zeros(n, int))
    elif case == "all_below_threshold":
        lg = rng.normal(0, 0.3, (n, 81))
    elif case == "over_100_one_class":        # 300 disjoint confident boxes of class 17: 100 per class kept
        lg = _confident(rng, n, np.where(np.arange(n) < 300, 17, 0))
        rois[:300] = _grid_boxes(300)
        dl[:] = 0
    elif case == "over_100_overall":          # 400 disjoint confident boxes of 4 classes: top 100 by score overall
        lg = _confident(rng, n, np.where(np.arange(n) < 400, 1 + np.arange(n) % 4, 0))
        rois[:400] = _grid_boxes(400)
        dl[:] = 0
    elif case == "zero_area_rois":            # padding rows of the proposal layer with confident logits, and clusters suppressed by NMS
        lg = _confident(rng, n, rng.integers(1, 4, n))
        rois[::3] = 0
    elif case == "outside_window":
        lg = _confident(rng, n, rng.integers(1, 81, n))
        rois = _boxes(rng, n, -0.3, 1.3)
    else:                                     # n < 1000
        n = {"n_1": 1, "n_37": 37, "n_999": 999}[case]
        lg = _confident(rng, n, rng.integers(0, 6, n), margin=3.0)
        return rois[:n], lg, dl[:n]
    return rois, lg, dl


@pytest.mark.parametrize("case", ["score_ties", "nan_logits", "all_background", "all_below_threshold", "over_100_one_class", "over_100_overall",
                                  "zero_area_rois", "outside_window", "n_1", "n_37", "n_999"])
def test_refine_crafted_inputs_bit_exact(nets, case):
    import torch
    bb, rpn, det = nets(1024)
    rois, lg, dl = (np.ascontiguousarray(x, np.float32) for x in _refine_case(case))
    t = [torch.from_numpy(x).cuda() for x in (rois, lg, dl)]
    det.refine(t[0].data_ptr(), t[1].data_ptr(), t[2].data_ptr(), rois.shape[0])
    n, dets = det.detections()
    rn, want, _ = ref.detection_layer(rois, lg, dl, _window(det))
    assert n == rn, (n, rn)
    assert np.array_equal(dets.view(np.uint32), want.view(np.uint32)), np.argwhere(dets.view(np.uint32) != want.view(np.uint32))[:5]
    if case in ("all_background", "all_below_threshold"):
        assert n == 0 and not dets.view(np.uint32).any()
    if case == "over_100_one_class":
        assert n == 100 and (dets[:, 4] == 17).all()
    if case == "over_100_overall":
        assert n == 100 and len(set(dets[:, 4].tolist())) == 4
    if case == "score_ties":
        assert n > 0 and 3 not in set(dets[:n, 4].tolist())


def _pixel_box(win, W, H, y1, x1, y2, x2):
    """the window-normalised box whose unmould is (about) the pixel box y1 x1 y2 x2"""
    n = np.array([y1 / (H - 1), x1 / (W - 1), (y2 - 1) / (H - 1), (x2 - 1) / (W - 1)])
    return (np.array([win[0], win[1], win[0], win[1]], np.float64) + n * np.array([win[2] - win[0], win[3] - win[1]] * 2)).astype(np.float32)


def _paste_case(case, S, W, H):
    rng = np.random.default_rng(zlib.crc32(case.encode()) + W)
    win = ref.window(S, W, H)
    dets = np.zeros((100, 6), np.float32)
    yy, xx = np.mgrid[0:28, 0:28]
    masks = np.stack([np.clip(0.5 + 0.4 * np.sin(yy / rng.uniform(2, 6) + xx / rng.uniform(2, 6) + rng.uniform(0, 6)), 0, 1)
                      for _ in range(100)]).astype(np.float32)
    masks[:, ::7, ::7] = 0.5                                  # values exactly 0.5 on grid points
    k = 0
    if case in ("edges", "hundred"):
        boxes = [(0, 0, H, W), (0, 0, H // 3, W // 2), (H // 2, W // 2, H, W), (0, W - 40, 60, W)]
    elif case == "tiny":                                      # 1-pixel boxes and boxes smaller than 28 px
        boxes = [(y, x, y + 1, x + 1) for y, x in zip(rng.integers(0, H - 1, 10), rng.integers(0, W - 1, 10))]
        boxes += [(y, x, y + h, x + w) for y, x, h, w in zip(rng.integers(0, H - 30, 10), rng.integers(0, W - 30, 10), rng.integers(2, 28, 10),
                                                             rng.integers(2, 28, 10))]
    elif case == "overlapping":
        boxes = [(50 + 10 * i, 60 + 15 * i, 250 + 10 * i, 300 + 15 * i) for i in range(12)]
    elif case == "zero_area":                                 # inverted in one axis: area <= 0 after rounding, dropped
        boxes = [(100, 100, 200, 200), (150, 150, 140, 300), (0, 0, 50, 50), (30, 300, 80, 290)]
    else:
        boxes = []
    if case == "hundred":
        c, s = rng.uniform(0, 1, (96, 2)), rng.uniform(0.02, 0.5, (96, 2))
        boxes += [(int(a * H), int(b * W), int(min(a + u, 1) * H) + 1, int(min(b + v, 1) * W) + 1) for (a, b), (u, v) in zip(c, s)]
    for y1, x1, y2, x2 in boxes:
        dets[k, :4] = _pixel_box(win, W, H, y1, x1, y2, x2)
        dets[k, 4] = 1 + k % 80
        dets[k, 5] = rng.uniform(0.6, 1.0)                    # above the default min_score: every detection with area is exported
        k += 1
    if case == "zero_area":
        dets[k, 4] = 0                                        # a class-0 row ends the list; the rows after it are not read
        dets[k + 1] = dets[0]
    return dets, masks


@pytest.mark.parametrize("case", ["edges", "tiny", "overlapping", "zero_area", "none", "hundred"])
@pytest.mark.parametrize("size", [(640, 480), (333, 517)])
def test_paste_crafted_inputs_bit_exact(nets, case, size):
    import torch
    bb, rpn, det = nets(1024)
    W, H = size
    dets, masks = _paste_case(case, 1024, W, H)
    td, tm = torch.from_numpy(dets).cuda(), torch.from_numpy(masks).cuda()
    det.paste(td.data_ptr(), tm.data_ptr(), W, H)
    img, cls, rois = det.idImage()
    rimg, rcls, rrois = ref.id_image(dets, masks, ref.window(1024, W, H), W, H)
    assert cls == rcls and rois == rrois
    assert np.array_equal(img, rimg), int((img != rimg).sum())
    if case == "none":
        assert not img.any() and cls == []
    if case == "hundred":
        assert len(cls) == 100
    if case == "overlapping":
        assert img[255, 300] == len(cls) or not ref.unmold_mask(masks[len(cls) - 1], tuple(rois[-1]), H, W)[255, 300]


def test_execute_is_deterministic(nets):
    bb, rpn, det = nets(1024)
    rgb = _frame()
    outs = []
    for _ in range(2):
        img, cls, rois = det.execute(rgb)
        n, dets = det.detections()
        outs.append((img, cls, rois, n, dets, det.masks(), det.headOutputs()[0]))
    a, b = outs
    assert np.array_equal(a[0], b[0]) and a[1] == b[1] and a[2] == b[2] and a[3] == b[3]
    for x, y in zip(a[4:], b[4:]):
        assert np.array_equal(x.view(np.uint32), y.view(np.uint32))
    # execute() is the forward of the fixture on the same frame
    assert np.array_equal(a[4].view(np.uint32), _forward_reference(det, 1024)[1].view(np.uint32))


def test_refine_rejects_bad_counts(nets):
    import torch
    import maskfusion_b200 as mfb
    bb, rpn, det = nets(256)
    t = torch.zeros(1001, 81, 4, device="cuda")
    for n in (0, -1, 1001):
        with pytest.raises(mfb.MFError, match="n = "):
            det.refine(t.data_ptr(), t.data_ptr(), t.data_ptr(), n)
