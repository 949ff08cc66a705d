"""numpy restatement of the Mask R-CNN region-proposal stage (csrc/mf_rpn.cu): pyramid anchors, the proposal layer and pyramid ROI Align
of matterport mrcnn (COCO InferenceConfig), with the written rules R-TOPK, R-NMS and R-ROILEVEL of DESIGN.md section 4.

Every float operation is float32 in the kernels' order (the CUDA file is compiled -fmad=false), so the GPU results are compared bit for bit."""
from __future__ import annotations

import numpy as np

f32 = np.float32
PRE_NMS, POST_NMS, NMS_THRESHOLD = 6000, 1000, f32(0.7)
BBOX_STD_DEV = np.array([0.1, 0.1, 0.2, 0.2], np.float32)


def pyramid_anchors(S: int) -> np.ndarray:
    """generate_pyramid_anchors(scales 32..512, ratios 0.5/1/2, strides 4..64, anchor stride 1) + norm_boxes, in float64, rounded to float32.
    Order: level P2..P6, then y, x, ratio."""
    ratios = np.array([0.5, 1.0, 2.0])
    out = []
    for lvl in range(5):
        n, scale, stride = S >> (lvl + 2), 32.0 * 2 ** lvl, 4.0 * 2 ** lvl
        h, w = scale / np.sqrt(ratios), scale * np.sqrt(ratios)
        cy = (np.arange(n) * stride)[:, None, None] + np.zeros((1, n, 3))
        cx = (np.arange(n) * stride)[None, :, None] + np.zeros((n, 1, 3))
        hh, ww = np.broadcast_to(h, (n, n, 3)), np.broadcast_to(w, (n, n, 3))
        out.append(np.stack([cy - 0.5 * hh, cx - 0.5 * ww, cy + 0.5 * hh, cx + 0.5 * ww], axis=-1).reshape(-1, 4))
    b = np.concatenate(out)
    return ((b - np.array([0.0, 0.0, 1.0, 1.0])) / (S - 1)).astype(np.float32)


def det_expf(x) -> np.ndarray:
    """R-EXP: Cody-Waite reduction + Cephes degree-6 polynomial, the device det_expf (csrc/mf_common.cuh)"""
    xin = np.asarray(x, np.float32)
    with np.errstate(invalid="ignore", over="ignore"):
        x = np.fmin(np.fmax(xin, f32(-87.0)), f32(88.0))
        n = np.floor(x * f32(1.44269504088896341) + f32(0.5))
        r = (x - n * f32(0.693359375)) - n * f32(-2.12194440e-4)
        p = f32(1.9875691500e-4)
        for c in (1.3981999507e-3, 8.3334519073e-3, 4.1665795894e-2, 1.6666665459e-1, 5.0000001201e-1):
            p = p * r + f32(c)
        y = (p * (r * r) + r) + f32(1.0)
        res = y * ((n.astype(np.int32) + 127).astype(np.uint32) << np.uint32(23)).view(np.float32)
        res = np.where(xin > f32(88.0), f32(np.inf), res)
        res = np.where(~(xin > f32(-87.0)), np.where(np.isnan(xin), xin, f32(0.0)), res)
    return res.astype(np.float32)


def scores(logits: np.ndarray) -> np.ndarray:
    """softmax over the two logits, foreground probability: e_i = exp(l_i - max), e1 / (e0 + e1)"""
    l0, l1 = logits[:, 0].astype(np.float32), logits[:, 1].astype(np.float32)
    m = np.where(l1 > l0, l1, l0)
    with np.errstate(invalid="ignore"):
        e0, e1 = det_expf(l0 - m), det_expf(l1 - m)
        return (e1 / (e0 + e1)).astype(np.float32)


def topk_order(s: np.ndarray, k: int) -> np.ndarray:
    """R-TOPK: descending score, ties by lower index, NaN last (-0 counts as +0)"""
    s = np.where(s == 0, f32(0.0), s).astype(np.float32)
    u = s.view(np.uint32).astype(np.uint64)
    ordk = np.where(u & 0x80000000, ~u & 0xFFFFFFFF, u | 0x80000000)
    ordk = np.where(np.isnan(s), 0, ordk)
    key = ((~ordk & 0xFFFFFFFF) << np.uint64(32)) | np.arange(s.shape[0], dtype=np.uint64)
    return np.argsort(key, kind="stable")[:k]


def apply_box_deltas(anchors: np.ndarray, deltas: np.ndarray) -> np.ndarray:
    """apply_box_deltas_graph in the upstream operation order, then clip_boxes_graph to [0, 0, 1, 1]"""
    a = anchors.astype(np.float32)
    d = deltas.astype(np.float32) * BBOX_STD_DEV
    with np.errstate(invalid="ignore", over="ignore"):
        h, w = a[:, 2] - a[:, 0], a[:, 3] - a[:, 1]
        cy, cx = a[:, 0] + f32(0.5) * h, a[:, 1] + f32(0.5) * w
        cy = cy + d[:, 0] * h
        cx = cx + d[:, 1] * w
        h = h * det_expf(d[:, 2])
        w = w * det_expf(d[:, 3])
        y1, x1 = cy - f32(0.5) * h, cx - f32(0.5) * w
        y2, x2 = y1 + h, x1 + w
    b = np.stack([y1, x1, y2, x2], axis=1)
    return np.fmax(np.fmin(b, f32(1.0)), f32(0.0)).astype(np.float32)


def _lesser(a, b):      # std::min
    return np.where(b < a, b, a)


def _greater(a, b):     # std::max
    return np.where(a < b, b, a)


def iou_row(b: np.ndarray, i: int, js: np.ndarray) -> np.ndarray:
    """R-NMS: TensorFlow's IoU of box i with boxes js (corners min/max-normalised, empty boxes overlap nothing)"""
    ymin, xmin = _lesser(b[:, 0], b[:, 2]), _lesser(b[:, 1], b[:, 3])
    ymax, xmax = _greater(b[:, 0], b[:, 2]), _greater(b[:, 1], b[:, 3])
    with np.errstate(invalid="ignore", divide="ignore", over="ignore"):
        area_i = (ymax[i] - ymin[i]) * (xmax[i] - xmin[i])
        area_j = (ymax[js] - ymin[js]) * (xmax[js] - xmin[js])
        iy0, ix0 = _greater(ymin[i], ymin[js]), _greater(xmin[i], xmin[js])
        iy1, ix1 = _lesser(ymax[i], ymax[js]), _lesser(xmax[i], xmax[js])
        inter = _greater(iy1 - iy0, f32(0.0)) * _greater(ix1 - ix0, f32(0.0))
        iou = inter / ((area_i + area_j) - inter)
    return np.where((area_i <= 0) | (area_j <= 0), f32(0.0), iou).astype(np.float32)


def nms(boxes: np.ndarray, max_out: int = POST_NMS, threshold=NMS_THRESHOLD) -> list:
    """greedy NMS over boxes already in R-TOPK order: j is suppressed by a kept i iff IoU > threshold; returns kept positions"""
    b = boxes.astype(np.float32)
    k = b.shape[0]
    suppressed = np.zeros(k, bool)
    keep = []
    for i in range(k):
        if suppressed[i]:
            continue
        keep.append(i)
        if len(keep) == max_out:
            break
        js = np.arange(i + 1, k)
        suppressed[js[iou_row(b, i, js) > threshold]] = True
    return keep


def proposal_layer(logits: np.ndarray, deltas: np.ndarray, anchors: np.ndarray):
    """ProposalLayer: -> (kept count, rois [1000, 4] normalised y1 x1 y2 x2, zero padded)"""
    n = logits.shape[0]
    order = topk_order(scores(logits), min(PRE_NMS, n))
    boxes = apply_box_deltas(anchors[order], deltas[order])
    keep = nms(boxes)
    rois = np.zeros((POST_NMS, 4), np.float32)
    rois[:len(keep)] = boxes[keep]
    return len(keep), rois


def area_scale(S: int):
    return f32(S * S / (224.0 * 224.0))


def roi_level(boxes: np.ndarray, S: int) -> np.ndarray:
    """R-ROILEVEL: t = (h*w) * fp32(S^2/224^2), level = 2 + [t >= 2^-3] + [t >= 2^-1] + [t >= 2]; NaN / degenerate -> 2"""
    b = boxes.astype(np.float32)
    with np.errstate(invalid="ignore", over="ignore"):
        t = ((b[:, 2] - b[:, 0]) * (b[:, 3] - b[:, 1])) * area_scale(S)
        return 2 + (t >= f32(0.125)).astype(int) + (t >= f32(0.5)).astype(int) + (t >= f32(2.0)).astype(int)


def roi_level_matterport(boxes: np.ndarray, S: int) -> np.ndarray:
    """PyramidROIAlign's own formula: min(5, max(2, 4 + round(log2(sqrt(h*w) / (224 / sqrt(S*S))))))"""
    b = boxes.astype(np.float64)
    r = np.sqrt((b[:, 2] - b[:, 0]) * (b[:, 3] - b[:, 1])) / (224.0 / S)
    return np.clip(4 + np.round(np.log2(r)).astype(int), 2, 5)


def to_bf16_bits(x: np.ndarray) -> np.ndarray:
    """float32 -> bf16 bit patterns, round to nearest even (finite inputs)"""
    u = np.ascontiguousarray(x, np.float32).view(np.uint32).astype(np.uint64)
    return ((u + 0x7FFF + ((u >> 16) & 1)) >> 16).astype(np.uint16)


def roi_align(levels, boxes: np.ndarray, pool: int, S: int) -> np.ndarray:
    """pyramid ROI Align: tf.image.crop_and_resize (bilinear, extrapolation 0) of each box on P(level); levels = [P2..P5] float32 (H, W, C)
    -> bf16 bit patterns [n, pool, pool, C], each value rounded once from the float32 interpolation"""
    b = boxes.astype(np.float32)
    C = levels[0].shape[2]
    out = np.zeros((b.shape[0], pool, pool, C), np.float32)
    lv = roi_level(b, S)
    steps = np.arange(pool).astype(np.float32)
    with np.errstate(invalid="ignore", over="ignore"):
        for r in range(b.shape[0]):
            F = levels[lv[r] - 2]
            H, W = F.shape[0], F.shape[1]
            y1, x1, y2, x2 = b[r]
            hs = ((y2 - y1) * f32(H - 1)) / f32(pool - 1)
            ws = ((x2 - x1) * f32(W - 1)) / f32(pool - 1)
            in_y = y1 * f32(H - 1) + steps * hs
            in_x = x1 * f32(W - 1) + steps * ws
            vy = (in_y >= 0) & (in_y <= f32(H - 1))
            vx = (in_x >= 0) & (in_x <= f32(W - 1))
            ty = np.where(vy, np.floor(in_y), 0).astype(int); by = np.where(vy, np.ceil(in_y), 0).astype(int)
            lx = np.where(vx, np.floor(in_x), 0).astype(int); rx = np.where(vx, np.ceil(in_x), 0).astype(int)
            yl = (in_y - ty.astype(np.float32))[:, None, None]
            xl = (in_x - lx.astype(np.float32))[None, :, None]
            tl, tr = F[ty][:, lx], F[ty][:, rx]
            bl, br = F[by][:, lx], F[by][:, rx]
            top = tl + (tr - tl) * xl
            bottom = bl + (br - bl) * xl
            v = top + (bottom - top) * yl
            out[r] = np.where((vy[:, None] & vx[None, :])[:, :, None], v, f32(0.0))
    return to_bf16_bits(out)
