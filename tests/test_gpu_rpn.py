"""Region-proposal stage on the GPU (csrc/mf_rpn.cu): RPN head, proposal layer and pyramid ROI Align on the backbone's P2..P6.

The 3x3 conv and the 1x1 heads are tensor-core GEMMs, checked against PyTorch fp32 with the backbone test's tolerances.  Everything after
the GEMMs is fixed-order IEEE fp32 and is compared bit for bit with the numpy restatement (tests/rpn_ref.py), run on the GPU's own head
outputs, anchors and P-level maps."""
from __future__ import annotations

import contextlib
import ctypes as C
import zlib

import numpy as np
import pytest

from tests import rpn_ref as ref

pytestmark = pytest.mark.gpu
f32 = np.float32


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


@pytest.fixture(scope="module")
def nets():
    """S -> (Backbone, RegionProposals) after one forward on a moulded synthetic 640x480 frame; both on torch's current stream"""
    import torch
    import maskfusion_b200 as mfb
    from maskfusion_b200.synth import SynthScene
    made = {}

    def get(S):
        if S not in made:
            bb = mfb.Backbone(S, seed=7, stream=torch.cuda.current_stream().cuda_stream)
            rgb, *_ = SynthScene(640, 480, n_objects=2, seed=5).render(0)
            rgba = torch.from_numpy(np.concatenate([rgb, np.full(rgb.shape[:2] + (1,), 255, np.uint8)], axis=2)).cuda()
            L = mfb.load_library()
            assert L.mf_backbone_mold(C.c_void_p(bb.h), C.c_void_p(rgba.data_ptr()), 640, 480) == 0
            bb.forward(L.mf_backbone_input_buffer(bb.h))
            rpn = mfb.RegionProposals(bb, seed=11)
            rpn.forward()
            torch.cuda.synchronize()
            made[S] = (bb, rpn)
        return made[S]

    yield get
    for bb, rpn in made.values():
        rpn.close()
        bb.close()


def _levels(bb):
    return [bb.download(4 + i) for i in range(4)]          # P2..P5, float32 (H, W, 256) holding the bf16 values


@pytest.mark.parametrize("S", [256, 1024])
def test_rpn_conv_matches_torch(nets, S):
    """S = 256: P5 (8x8) and P6 (4x4) take the im2col path; S = 1024: every level the implicit 3x3 GEMM"""
    import torch
    import torch.nn.functional as F
    bb, rpn = nets(S)
    cw, cb, _, _ = rpn.weights()
    w = torch.from_numpy(cw).cuda().permute(0, 3, 1, 2).contiguous()
    b = torch.from_numpy(cb).cuda()
    with _no_tf32():
        for lvl in range(5):
            x = torch.from_numpy(bb.download(4 + lvl)).cuda().permute(2, 0, 1)[None]
            want = torch.relu(F.conv2d(x, w, b, padding=1))[0].permute(1, 2, 0)
            got = torch.from_numpy(rpn.convOutput(lvl)).cuda()
            assert got.shape == (S >> (lvl + 2), S >> (lvl + 2), 512)
            assert not torch.isnan(got).any(), lvl
            err, scale = (got - want).abs().max().item(), want.abs().max().item()
            assert scale > 1e-2, (lvl, "degenerate conv output")
            assert err <= 2.0 ** -7 * max(scale, 1.0), (lvl, err, scale)


@pytest.mark.parametrize("S", [256, 1024])
def test_rpn_heads_fp32_match_torch(nets, S):
    import torch
    bb, rpn = nets(S)
    _, _, hw, hb = rpn.weights()
    X = torch.from_numpy(np.concatenate([rpn.convOutput(l).reshape(-1, 512) for l in range(5)])).cuda()
    with _no_tf32():
        want = X @ torch.from_numpy(hw).cuda().t() + torch.from_numpy(hb).cuda()[None, :]
    lg, dl = rpn.headOutputs()
    got = torch.from_numpy(np.concatenate([lg.reshape(-1, 6), dl.reshape(-1, 12)], axis=1)).cuda()
    assert got.shape == want.shape == (rpn.A // 3, 18)
    err, scale = (got - want).abs().max().item(), want.abs().max().item()
    assert err <= 1e-4 * max(scale, 1.0), (err, scale)
    # damped head layers: boxes stay near their anchors, and the scores are spread out rather than saturated at 0 / 1
    assert 0.005 < float(np.abs(dl).mean()) < 1.0, float(np.abs(dl).mean())
    s = ref.scores(lg)
    assert ((s > 0.01) & (s < 0.99)).mean() > 0.5, np.percentile(s, [1, 50, 99])


@pytest.mark.parametrize("S", [256, 1024])
def test_proposals_bit_exact(nets, S):
    bb, rpn = nets(S)
    rpn.forward()
    anc = rpn.anchors()
    assert np.array_equal(anc.view(np.uint32), ref.pyramid_anchors(S).view(np.uint32))
    lg, dl = rpn.headOutputs()
    n, rois = rpn.proposals()
    rn, rrois = ref.proposal_layer(lg, dl, anc)
    assert n == rn and n > 0, (n, rn)
    assert np.array_equal(rois.view(np.uint32), rrois.view(np.uint32)), np.argwhere(rois.view(np.uint32) != rrois.view(np.uint32))[:5]


def _boxes(rng, n, lo=0.0, hi=1.0, smin=0.02, smax=0.3):
    c = rng.uniform(lo, hi, (n, 2)); s = rng.uniform(smin, smax, (n, 2))
    return np.concatenate([c - s / 2, c + s / 2], axis=1).astype(np.float32)


def _crafted(case):
    rng = np.random.default_rng(zlib.crc32(case.encode()))
    if case == "ties_at_topk_boundary":       # 6 distinct scores over 20 000 anchors: the 6000th falls inside a tie group
        n = 20000
        lg = np.stack([np.zeros(n), rng.integers(0, 6, n) * 0.5], 1)
        return lg, rng.normal(0, 1, (n, 4)), _boxes(rng, n)
    if case == "ties_all_selected":           # 3 distinct scores, n < 6000
        n = 5000
        lg = np.stack([np.full(n, 0.25), rng.integers(-1, 2, n).astype(float)], 1)
        return lg, rng.normal(0, 1, (n, 4)), _boxes(rng, n)
    if case == "degenerate_boxes":            # zero-area and inverted anchors among normal ones
        n = 7000
        a = _boxes(rng, n)
        a[0::3, 2] = a[0::3, 0]                                      # zero height
        a[1::3] = a[1::3][:, [2, 3, 0, 1]]                           # inverted
        d = rng.normal(0, 1, (n, 4)); d[::5] = 0
        return np.stack([np.zeros(n), rng.normal(0, 1, n)], 1), d, a
    if case == "duplicates_one_kept":         # every box suppresses every other: one kept, 999 zero rows
        n = 3000
        return np.stack([np.zeros(n), rng.normal(0, 1, n)], 1), np.zeros((n, 4)), np.repeat(_boxes(rng, 1), n, axis=0)
    if case == "clusters_fewer_than_1000":    # 400 distinct boxes x 12 copies
        n = 4800
        return np.stack([np.zeros(n), rng.normal(0, 1, n)], 1), np.zeros((n, 4)), np.repeat(_boxes(rng, 400, smin=0.05), 12, axis=0)
    n = {"n_4099_with_nan": 4099, "n_1": 1, "n_257": 257, "n_6001": 6001}[case]
    lg = np.stack([np.zeros(n), rng.normal(0, 2, n)], 1)
    if n > 100:
        lg[rng.choice(n, 50, replace=False), 1] = np.nan           # NaN scores rank last
    return lg, rng.normal(0, 1, (n, 4)), _boxes(rng, n, -0.1, 1.1)


@pytest.mark.parametrize("case", ["ties_at_topk_boundary", "ties_all_selected", "degenerate_boxes", "duplicates_one_kept", "clusters_fewer_than_1000",
                                  "n_4099_with_nan", "n_1", "n_257", "n_6001"])
def test_propose_crafted_inputs_bit_exact(nets, case):
    import torch
    bb, rpn = nets(1024)
    lg, dl, an = (np.ascontiguousarray(x, np.float32) for x in _crafted(case))
    n = lg.shape[0]
    t = [torch.from_numpy(x).cuda() for x in (lg, dl, an)]
    rpn.propose(t[0].data_ptr(), t[1].data_ptr(), t[2].data_ptr(), n)
    got_n, rois = rpn.proposals()
    want_n, want = ref.proposal_layer(lg, dl, an)
    assert got_n == want_n, (got_n, want_n)
    assert np.array_equal(rois.view(np.uint32), want.view(np.uint32))
    if case == "duplicates_one_kept":
        assert got_n == 1 and not rois[1:].view(np.uint32).any()
    if case == "clusters_fewer_than_1000":
        assert got_n <= 400 and not rois[got_n:].view(np.uint32).any()


def test_propose_rejects_bad_counts(nets):
    import torch
    import maskfusion_b200 as mfb
    bb, rpn = nets(256)
    t = torch.zeros(rpn.A + 1, 4, device="cuda")
    for n in (0, -1, rpn.A + 1):
        with pytest.raises(mfb.MFError, match="n_anchors"):
            rpn.propose(t.data_ptr(), t.data_ptr(), t.data_ptr(), n)


def _threshold_boxes(S):
    """for each level threshold B: boxes whose t = (h*w) * fp32(S^2/224^2) is the largest value below B, exactly B and the smallest value
    above B that a float h*w can produce (h*w lies on a fixed float grid, so one ulp below/above is not reachable at every S)"""
    sc = ref.area_scale(S)
    out = []
    for B in (f32(0.125), f32(0.5), f32(2.0)):
        cand, ts = [], []
        for h in np.linspace(0.2, 0.9, 64):
            y1 = f32(0.05); y2 = f32(y1 + f32(h)); hh = f32(y2 - y1)
            x1 = f32(0.02); x2c = f32(x1 + f32(B / (float(sc) * float(hh))))
            x2 = (x2c.astype(np.float64) + np.arange(-100, 101) * float(np.spacing(x2c))).astype(np.float32)
            ts.append((hh * (x2 - x1)) * sc)
            cand.append(np.stack([np.full_like(x2, y1), np.full_like(x2, x1), np.full_like(x2, y2), x2], axis=1))
        t, cand = np.concatenate(ts), np.concatenate(cand)
        below, above = np.max(t[t < B]), np.min(t[t > B])
        assert below == np.nextafter(B, f32(0)) or below == np.nextafter(np.nextafter(B, f32(0)), f32(0)), (B, below)
        assert above == np.nextafter(B, f32(4)), (B, above)
        assert (t == B).any(), B
        boxes = cand[[np.argmax(t == below), np.argmax(t == B), np.argmax(t == above)]]
        lv = ref.roi_level(boxes, S)
        assert lv[1] == lv[2] == lv[0] + 1, (B, lv)
        out.append(boxes)
    return np.concatenate(out)


def _roi_align_gpu(bb, boxes, pool):
    import torch
    import maskfusion_b200 as mfb
    n = boxes.shape[0]
    out = torch.full((max(n, 1), pool, pool, 256), 0x7FC1, dtype=torch.int16, device="cuda")    # NaN pattern: unwritten values show
    tb = torch.from_numpy(np.ascontiguousarray(boxes, np.float32).reshape(-1, 4)).cuda()
    mfb.roi_align(bb, tb.data_ptr(), n, pool, out.data_ptr())
    torch.cuda.synchronize()
    return out.cpu().numpy().view(np.uint16)


@pytest.mark.parametrize("S", [256, 1024])
def test_forward_roi_align_bit_exact(nets, S):
    bb, rpn = nets(S)
    rpn.forward()
    n, rois = rpn.proposals()
    want = ref.roi_align(_levels(bb), rois, 7, S)
    got = rpn.pooled(raw=True)
    assert got.shape == (1000, 7, 7, 256)
    assert np.array_equal(got, want)               # every pyramid level is covered by the crafted boxes below


@pytest.mark.parametrize("pool", [7, 14])
def test_roi_align_crafted_boxes_bit_exact(nets, pool):
    bb, rpn = nets(1024)
    S = 1024
    levels = _levels(bb)
    special = np.array([[-0.2, -0.1, 0.5, 0.6], [1.1, 1.2, 1.5, 1.6], [-0.5, -0.5, -0.1, -0.1], [0.3, -0.4, 0.9, 0.2], [0.5, 0.5, 1.3, 1.4],
                        [0.3, 0.3, 0.3, 0.3], [0.7, 0.2, 0.7, 0.6], [0.8, 0.8, 0.2, 0.3], [0.0, 0.0, 1.0, 1.0]], np.float32)
    thr = _threshold_boxes(S)
    rng = np.random.default_rng(pool)
    c, s = rng.uniform(-0.2, 1.2, (1000, 2)), np.exp(rng.uniform(np.log(0.005), 0.0, (1000, 2)))
    many = np.concatenate([c - s / 2, c + s / 2], axis=1).astype(np.float32)          # partly outside, every pyramid level
    for boxes in (np.concatenate([special, thr]), thr[4:5], many):
        got = _roi_align_gpu(bb, boxes, pool)
        assert np.array_equal(got, ref.roi_align(levels, boxes, pool, S)), boxes.shape
    assert set(ref.roi_level(many, S)) == {2, 3, 4, 5}
    empty = _roi_align_gpu(bb, np.zeros((0, 4), np.float32), pool)
    assert (empty == 0x7FC1).all()


def test_forward_is_deterministic(nets):
    import maskfusion_b200 as mfb
    bb, rpn = nets(1024)
    rpn.forward()
    n0, r0 = rpn.proposals(); p0 = rpn.pooled(raw=True)
    bb.forward(mfb.load_library().mf_backbone_input_buffer(bb.h))
    rpn.forward()
    n1, r1 = rpn.proposals(); p1 = rpn.pooled(raw=True)
    assert n0 == n1 and np.array_equal(r0.view(np.uint32), r1.view(np.uint32)) and np.array_equal(p0, p1)


def test_rpn_leaves_backbone_table_alone(nets):
    import maskfusion_b200 as mfb
    bb, rpn = nets(256)
    assert len(bb.layers()) == 1 + 33 * 3 + 4 + 8
    bb.forward(mfb.load_library().mf_backbone_input_buffer(bb.h))
    rpn.forward()
    assert bb.numGemms() == 112
