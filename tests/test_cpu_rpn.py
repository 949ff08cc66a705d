"""The numpy restatement of the region-proposal stage (tests/rpn_ref.py) on its own: anchors, exp, bf16 rounding, NMS against torchvision and the
ROI level rule against matterport's formula.  The GPU kernels are compared with this restatement in tests/test_gpu_rpn.py."""
from __future__ import annotations

import numpy as np
import pytest

from tests import rpn_ref as ref


@pytest.mark.parametrize("S,count", [(256, 16368), (1024, 261888)])
def test_anchor_count_and_order(S, count):
    a = ref.pyramid_anchors(S)
    assert a.shape == (count, 4) and a.dtype == np.float32
    # order (level, y, x, ratio): within a pixel the ratio 0.5 / 1 / 2 anchors are tall -> square -> wide, same centre
    first = a[:3].astype(np.float64) * (S - 1) + [0, 0, 1, 1]
    h, w = first[:, 2] - first[:, 0], first[:, 3] - first[:, 1]
    assert np.allclose(h, [32 * 2 ** 0.5, 32, 32 / 2 ** 0.5]) and np.allclose(w, [32 / 2 ** 0.5, 32, 32 * 2 ** 0.5])
    # x runs fastest after the ratio: pixel (0, 1) of P2 is 4 pixels (stride) to the right of pixel (0, 0)
    assert np.allclose((a[3:6] - a[0:3]).astype(np.float64) * (S - 1), [[0, 4, 0, 4]] * 3)
    # level boundaries: P3 starts after (S/4)^2 * 3 anchors with the 64-pixel square anchor at ratio 1
    p3 = 3 * (S // 4) ** 2
    sq = a[p3 + 1].astype(np.float64) * (S - 1) + [0, 0, 1, 1]
    assert np.allclose([sq[2] - sq[0], sq[3] - sq[1]], [64, 64])


def test_anchor_hand_computed():
    """S = 1024, P3 (stride 8, scale 64), y = 5, x = 7, ratio 2: h = 64 / sqrt 2, w = 64 sqrt 2, centre (40, 56)"""
    a = ref.pyramid_anchors(1024)
    idx = 3 * 256 * 256 + (5 * 128 + 7) * 3 + 2
    half_h, half_w = 22.627416997969522, 45.254833995939045
    want = np.array([(40 - half_h) / 1023, (56 - half_w) / 1023, (40 + half_h - 1) / 1023, (56 + half_w - 1) / 1023], np.float32)
    assert np.array_equal(a[idx], want), (a[idx], want)


def test_det_expf_matches_oracle(oracle):
    L = oracle.lib()
    xs = np.concatenate([np.linspace(-90, 90, 2001), np.random.default_rng(0).normal(0, 3, 2000)]).astype(np.float32)
    got = ref.det_expf(xs)
    want = np.array([L.orc_expf(float(x)) for x in xs], np.float32)
    assert np.array_equal(got.view(np.uint32), want.view(np.uint32))


def test_bf16_rounding_matches_torch():
    import torch
    x = (np.random.default_rng(1).normal(0, 10, 100000)).astype(np.float32)
    x[:4] = [0.0, -0.0, 1.00390625, 1.01171875]           # ties to even, both directions
    want = torch.from_numpy(x).to(torch.bfloat16).view(torch.int16).numpy().view(np.uint16)
    assert np.array_equal(ref.to_bf16_bits(x), want)


def _random_boxes(rng, n):
    c = rng.uniform(0, 1, (n, 2)); s = rng.uniform(0.02, 0.3, (n, 2))
    return np.concatenate([c - s / 2, c + s / 2], axis=1).astype(np.float32)


@pytest.mark.parametrize("seed", [0, 1, 2])
def test_nms_matches_torchvision(seed):
    import torch
    import torchvision
    rng = np.random.default_rng(seed)
    boxes = _random_boxes(rng, 3000)
    sc = rng.permutation(3000).astype(np.float32)                   # distinct scores: no ties
    order = np.argsort(-sc, kind="stable")
    keep = ref.nms(boxes[order], max_out=10 ** 9)
    tb = torch.from_numpy(boxes[:, [1, 0, 3, 2]].copy())             # torchvision: x1 y1 x2 y2
    want = torchvision.ops.nms(tb, torch.from_numpy(sc), 0.7).numpy()
    assert 100 < len(keep) < 3000
    assert np.array_equal(order[keep], want)


def test_nms_stops_at_max_and_pads():
    rng = np.random.default_rng(3)
    boxes = _random_boxes(rng, 8000)
    logits = np.stack([np.zeros(8000), rng.normal(0, 1, 8000)], 1).astype(np.float32)
    n, rois = ref.proposal_layer(logits, np.zeros((8000, 4), np.float32), boxes)
    assert n == 1000 and rois.shape == (1000, 4)
    dup = np.repeat(np.clip(boxes[:1], 0, 1), 50, axis=0)
    n1, rois1 = ref.proposal_layer(np.zeros((50, 2), np.float32), np.zeros((50, 4), np.float32), dup)
    assert n1 == 1 and np.allclose(rois1[0], dup[0], atol=1e-6) and not rois1[1:].any()


def test_roi_level_rule_matches_matterport_away_from_boundaries():
    rng = np.random.default_rng(4)
    for S in (256, 1024):
        b = _random_boxes(rng, 20000) * np.float32(rng.uniform(0.1, 3.0))
        t = ((b[:, 2] - b[:, 0]).astype(np.float64) * (b[:, 3] - b[:, 1])) * S * S / 224.0 ** 2
        far = np.min(np.abs(np.log2(t)[:, None] - np.log2([0.125, 0.5, 2.0])[None, :]), axis=1) > 1e-4
        assert far.sum() > 19000
        assert np.array_equal(ref.roi_level(b, S)[far], ref.roi_level_matterport(b, S)[far])
