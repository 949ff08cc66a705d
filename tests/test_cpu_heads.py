"""The numpy restatement of the detection heads (tests/heads_ref.py) on its own: per-class NMS against torchvision, the mask resize against
scipy.ndimage.zoom (the pin of R-RESIZE), unmould on boxes worked out by hand, the restated export path against api.generate_id_image, and
the input mould's resample against scipy.ndimage.zoom (the pin of R-MOLD).  The GPU kernels are compared with this restatement in
tests/test_gpu_heads.py and tests/test_gpu_cnn.py."""
from __future__ import annotations

import numpy as np
import pytest

from tests import heads_ref as ref
from tests import rpn_ref

f32 = np.float32


def test_class_nms_matches_torchvision_batched_nms():
    import torch
    from torchvision.ops import batched_nms, box_iou
    rng = np.random.default_rng(3)
    n = 600
    c, s = rng.uniform(0, 1, (n, 2)), rng.uniform(0.05, 0.3, (n, 2))
    boxes = np.concatenate([c - s / 2, c + s / 2], axis=1).astype(np.float32)
    scores = rng.permutation(np.linspace(0.71, 0.99, n)).astype(np.float32)           # tie-free
    classes = rng.integers(1, 6, n)
    iou = box_iou(*[torch.from_numpy(boxes[:, [1, 0, 3, 2]]).double()] * 2).numpy()
    near = (classes[:, None] == classes[None, :]) & (np.abs(iou - 0.3) < 1e-3)
    np.fill_diagonal(near, False)
    away = ~near.any(1)                                        # drop boxes of a same-class pair near the threshold
    boxes, scores, classes = boxes[away], scores[away], classes[away]
    n = boxes.shape[0]
    assert n > 500
    xyxy = torch.from_numpy(boxes[:, [1, 0, 3, 2]]).double()
    kept, removed = ref.class_nms(boxes, scores, classes, np.arange(n))
    want = batched_nms(xyxy, torch.from_numpy(scores).double(), torch.from_numpy(classes), 0.3).numpy()
    assert removed > 0 and sorted(kept.tolist()) == sorted(want.tolist())


def _zoom(m, h, w):
    """skimage.transform.resize(m, (h, w), order=1, mode='constant', anti_aliasing=False) as skimage >= 0.19 computes it"""
    import scipy.ndimage as ndi
    return ndi.zoom(m, (1 / (28 / h), 1 / (28 / w)), order=1, mode="grid-constant", cval=0.0, grid_mode=True)


def test_resize_matches_scipy_zoom():
    rng = np.random.default_rng(5)
    smooth = np.clip(0.5 + 0.5 * np.sin(np.mgrid[0:28, 0:28][0] / 3.0) * np.cos(np.mgrid[0:28, 0:28][1] / 4.0), 0, 1).astype(np.float32)
    half = rng.uniform(0, 1, (28, 28)).astype(np.float32)
    half[::3, ::2] = 0.5                                       # values exactly 0.5 on grid points
    masks = [rng.uniform(0, 1, (28, 28)).astype(np.float32), smooth, half]
    sides = [1, 2, 3, 7, 13, 14, 27, 28, 29, 41, 55, 56, 57, 100, 199, 333, 480, 600]
    differ = total = 0
    for m in masks:
        for h in sides:
            for w in sides[::3] + [600]:
                got, want = ref.resize_mask(m, h, w), _zoom(m, h, w)
                assert want.shape == (h, w) and want.dtype == np.float32
                ulps = np.abs(got.view(np.int32).astype(np.int64) - want.view(np.int32).astype(np.int64))
                assert ulps.max() <= 1, (h, w, ulps.max())
                assert np.array_equal(got >= f32(0.5), want >= f32(0.5)), (h, w)
                differ += int((ulps > 0).sum()); total += ulps.size
    print(f"R-RESIZE: {differ} of {total} float32 values differ from scipy.ndimage.zoom by 1 ulp, none by more; threshold decisions identical")
    assert (ref.resize_mask(masks[2], 28, 28) == masks[2]).all()      # the identity resize reproduces the grid, 0.5 included


@pytest.mark.parametrize("W,H,S", [(640, 480, 256), (640, 480, 1024), (1280, 720, 1024), (320, 240, 1024), (480, 640, 1024), (641, 479, 1024),
                                   (7, 5, 64), (100, 37, 64)])
def test_mold_resize_matches_scipy_zoom(W, H, S):
    """R-MOLD's resample, truncated to uint8, against scipy.ndimage.zoom (skimage >= 0.19's resize(order=1, mode='constant',
    preserve_range=True)) of the same float64 image: zero differing bytes, at sizes whose scale is not an integer ratio too"""
    import scipy.ndimage as ndi
    _, nw, nh, ox, oy = ref.mold_geometry(S, W, H)
    for kind in ref.MOLD_KINDS:
        rgba = ref.mold_test_image(kind, W, H, seed=W + H)
        bits, box = ref.mold_input(rgba, S)
        want = ndi.zoom(rgba[..., :3].astype(np.float64), (nh / H, nw / W, 1), order=1, mode="grid-constant", cval=0.0, grid_mode=True)
        assert want.shape == box.shape == (nh, nw, 3)
        assert int((want.astype(np.uint8) != box).sum()) == 0, (kind, W, H, S)
        # the letter box and only it holds the resized image; the padding is the uint8 value 0 minus the mean pixel
        pad = ref.bf16_bits(-np.array(ref.MEAN_PIXEL, np.float32))
        inside = np.zeros((S, S), bool)
        inside[oy:oy + nh, ox:ox + nw] = True
        assert (bits[~inside] == pad).all()
        assert np.array_equal(bits[inside].reshape(nh, nw, 3), ref.bf16_bits((box.astype(np.float32) - np.array(ref.MEAN_PIXEL)).astype(np.float32)))


def test_mold_rule_worked_by_hand():
    """a flat 200 image at 640 x 480 -> S = 1024: letter box 1024 x 768 at y = 128, zoom 640 / 1024 = 0.625.  Resized sample 0 reads
    c = 0.5 * 0.625 - 0.5 = -0.1875: taps -1 (outside, 0) and 0 with weights 0.1875 and 0.8125, so the first and last row and column
    blend with 0 (200 * 0.8125 = 162.5 -> 162, a corner 200 * 0.8125^2 = 132.03 -> 132) and the rest is 200.  In bf16: 76.3 -> 76.5,
    38.3 -> 38.25, 8.3 -> 8.3125, the padding -123.7 -> -123.5"""
    rgba = np.full((480, 640, 4), 200, np.uint8)
    bits, box = ref.mold_input(rgba, 1024)
    r = box[..., 0]
    assert r[0, 0] == r[0, -1] == r[-1, 0] == r[-1, -1] == 132
    assert (r[0, 1:-1] == 162).all() and (r[-1, 1:-1] == 162).all() and (r[1:-1, 0] == 162).all() and (r[1:-1, -1] == 162).all()
    assert (box[1:-1, 1:-1] == 200).all()
    f = (bits[..., 0].astype(np.uint32) << 16).view(np.float32)
    assert f[128 + 5, 5] == 76.5 and f[128, 5] == 38.25 and f[128, 0] == 8.3125
    assert (f[:128] == -123.5).all() and (f[128 + 768:] == -123.5).all()


def test_unmold_boxes_worked_by_hand():
    # a square 5 x 5 image fills the 256 x 256 input: window (0, 0, 1, 1), denorm multiplies by 4 and adds (0, 0, 1, 1)
    win = ref.window(256, 5, 5)
    assert win.tolist() == [0.0, 0.0, 1.0, 1.0]
    dets = np.zeros((100, 6), np.float32)
    dets[0] = [0.125, 0.375, 0.625, 0.875, 3, 0.9]           # 0.5 -> 0, 1.5 -> 2, 3.5 -> 4, 4.5 -> 4: half to even
    dets[1] = [0.5, 0.5, 0.25, 0.9, 4, 0.9]                  # y2 = 0.25 * 4 + 1 = 2 = y1: zero area, dropped
    dets[2] = [0.0, 0.0, 1.0, 1.0, 5, 0.8]                   # the whole image: (0, 0, 5, 5), on every edge
    u = ref.unmold(dets, win, 5, 5)
    assert [r[:5] for r in u] == [(0, 0, 2, 4, 4), (2, 0, 0, 5, 5)]
    # a 5 x 3 (W x H) image at 256: scale 51.2, 256 x 154 at y offset 51; window (51/255, 0, 204/255, 1); the window's corners map to the image's
    win = ref.window(256, 5, 3)
    assert np.array_equal(win, np.array([51 / 255, 0, 204 / 255, 1], np.float64).astype(np.float32))
    dets = np.zeros((100, 6), np.float32)
    dets[0] = [win[0], win[1], win[2], win[3], 1, 0.7]
    assert [r[1:5] for r in ref.unmold(dets, win, 5, 3)] == [(0, 0, 3, 5)]


def _random_detections(rng, S, W, H, n):
    win = ref.window(S, W, H)
    dets = np.zeros((100, 6), np.float32)
    c, s = rng.uniform(0, 1, (n, 2)), rng.uniform(0.01, 0.6, (n, 2))
    b = np.clip(np.concatenate([c - s / 2, c + s / 2], axis=1), 0, 1)
    dets[:n, :4] = np.array([win[0], win[1], win[0], win[1]]) + b * np.array([win[2] - win[0], win[3] - win[1]] * 2)
    dets[:n, 4] = rng.integers(1, 81, n)
    dets[:n, 5] = rng.uniform(0.5, 1.0, n)
    masks = rng.uniform(0, 1, (100, 28, 28)).astype(np.float32)
    masks = (masks + np.roll(masks, 1, 1) + np.roll(masks, 1, 2)) / 3            # some spatial structure
    return dets, masks.astype(np.float32), win


@pytest.mark.parametrize("export", ["default", "filtered"])
def test_export_path_matches_generate_id_image(product_lib, export):
    from maskfusion_b200 import api
    rng = np.random.default_rng(11)
    W, H = 160, 120
    dets, masks, win = _random_detections(rng, 256, W, H, 40)
    if export == "default":
        args = (0.55, (), ())
    else:
        c = int(dets[0, 4])
        special = [200 + i for i in range(81)]
        special[c] = 9; special[9] = c
        args = (0.7, tuple(int(x) for x in dets[:20, 4]), tuple(special))
    img, cls, rois = ref.id_image(dets, masks, win, W, H, *args)
    want = api.generate_id_image(ref.unmolded_result(dets, masks, win, W, H), *args)
    assert cls == want[1] and rois == want[2]
    assert np.array_equal(img, want[0])
    assert len(set(np.unique(img).tolist()) - {0}) >= 2


def test_sigmoid_and_softmax_rules():
    x = np.array([-100, -3, 0, 3, 100], np.float32)
    assert np.array_equal(ref.sigmoid(x), (f32(1) / (f32(1) + rpn_ref.det_expf(-x))).astype(np.float32))
    assert ref.sigmoid(np.float32(0.0)) == f32(0.5)
    lg = np.zeros((3, 81), np.float32)
    lg[0, 3] = lg[0, 4] = 5.0                                  # tie: the lower class index
    lg[1, 7] = np.nan                                          # any NaN logit: every p NaN -> class 0
    lg[2, 0] = np.nan                                          # NaN first
    cls, p = ref.softmax_argmax(lg)
    assert cls.tolist() == [3, 0, 0] and np.isnan(p[1:]).all()
