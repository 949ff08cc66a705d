"""numpy restatement of the Mask R-CNN detection heads after their GEMMs (csrc/mf_heads.cu): the detection layer, the mask select, unmould
and generate_id_image of matterport mrcnn (COCO InferenceConfig), with the written rules R-SOFTMAX, R-DETNMS, R-UNMOLD, R-RESIZE and R-SIGMOID
of DESIGN.md section 4; and the network's input mould (csrc/mf_cnn.cu k_mold_input), rule R-MOLD.

Float operations are float32 in the kernels' order (the CUDA file is compiled -fmad=false), float64 where R-UNMOLD and R-RESIZE say so, so the
GPU results are compared bit for bit."""
from __future__ import annotations

import numpy as np

from tests import rpn_ref
from tests.rpn_ref import det_expf, iou_row, f32

NUM_CLASSES, MAX_DET, MIN_CONFIDENCE, NMS_THRESHOLD, MASK = 81, 100, f32(0.7), f32(0.3), 28


def mold_geometry(S: int, W: int, H: int):
    """mf_backbone_mold's letter box: scale = min(S/W, S/H) in float32, new size lroundf(W * scale), centred (integer halves)"""
    scale = min(f32(S) / f32(W), f32(S) / f32(H))
    nw, nh = int(np.floor(np.float64(f32(W) * scale) + 0.5)), int(np.floor(np.float64(f32(H) * scale) + 0.5))
    return scale, nw, nh, (S - nw) // 2, (S - nh) // 2


def window(S: int, W: int, H: int) -> np.ndarray:
    """norm_boxes of the pixel window (y1, x1, y2, x2) = (offy, offx, offy + newH, offx + newW): (w - (0, 0, 1, 1)) / (S - 1) in float64,
    then float32"""
    _, nw, nh, ox, oy = mold_geometry(S, W, H)
    return ((np.array([oy, ox, oy + nh, ox + nw], np.float64) - [0, 0, 1, 1]) / (S - 1)).astype(np.float32)


def softmax_argmax(logits: np.ndarray):
    """R-SOFTMAX: m = sequential max (a NaN after the first logit is skipped), e_i = det_expf(l_i - m), sum in class order from 0,
    p_i = e_i / sum; class = first index of the largest p (strict >); any NaN logit makes every p NaN -> class 0"""
    l = logits.astype(np.float32)
    n = l.shape[0]
    with np.errstate(invalid="ignore", over="ignore"):
        m = l[:, 0].copy()
        for c in range(1, NUM_CLASSES):
            m = np.where(l[:, c] > m, l[:, c], m)
        s = np.zeros(n, np.float32)
        for c in range(NUM_CLASSES):
            s = (s + det_expf(l[:, c] - m)).astype(np.float32)
        best = np.zeros(n, np.int64)
        pbest = (det_expf(l[:, 0] - m) / s).astype(np.float32)
        for c in range(1, NUM_CLASSES):
            p = (det_expf(l[:, c] - m) / s).astype(np.float32)
            up = p > pbest
            best = np.where(up, c, best); pbest = np.where(up, p, pbest)
    return best, pbest


def apply_box_deltas_window(rois: np.ndarray, deltas: np.ndarray, win: np.ndarray) -> np.ndarray:
    """decode_box: apply_box_deltas_graph (deltas x BBOX_STD_DEV) then clip_boxes_graph to the window: max(min(v, hi), lo)"""
    b = _decode(rois, deltas)
    lo = np.array([win[0], win[1], win[0], win[1]], np.float32); hi = np.array([win[2], win[3], win[2], win[3]], np.float32)
    return np.fmax(np.fmin(b, hi), lo).astype(np.float32)


def _decode(anchors: np.ndarray, deltas: np.ndarray) -> np.ndarray:
    a = anchors.astype(np.float32)
    d = deltas.astype(np.float32) * rpn_ref.BBOX_STD_DEV
    with np.errstate(invalid="ignore", over="ignore"):
        h, w = a[:, 2] - a[:, 0], a[:, 3] - a[:, 1]
        cy, cx = a[:, 0] + f32(0.5) * h, a[:, 1] + f32(0.5) * w
        cy = cy + d[:, 0] * h
        cx = cx + d[:, 1] * w
        h = h * det_expf(d[:, 2])
        w = w * det_expf(d[:, 3])
        y1, x1 = cy - f32(0.5) * h, cx - f32(0.5) * w
        y2, x2 = y1 + h, x1 + w
    return np.stack([y1, x1, y2, x2], axis=1).astype(np.float32)


def _score_key(s: np.ndarray) -> np.ndarray:
    """~ord(score) as uint64 (R-TOPK's order map: -0 is +0, NaN last)"""
    s = np.where(s == 0, f32(0.0), s).astype(np.float32)
    u = s.view(np.uint32).astype(np.uint64)
    o = np.where(u & 0x80000000, ~u & 0xFFFFFFFF, u | 0x80000000)
    o = np.where(np.isnan(s), 0, o)
    return ~o & np.uint64(0xFFFFFFFF)


def class_nms(boxes: np.ndarray, scores: np.ndarray, classes: np.ndarray, cand: np.ndarray, max_per_class=MAX_DET, threshold=NMS_THRESHOLD):
    """R-DETNMS: per class, candidates in (score descending, lower ROI index) order; a candidate is suppressed by a kept one of its class
    iff IoU > threshold; at most max_per_class kept per class.  Returns the kept ROI indices (unordered) and the number NMS removed"""
    kept, removed = [], 0
    for c in np.unique(classes[cand]):
        idx = cand[classes[cand] == c]
        idx = idx[np.lexsort((idx, _score_key(scores[idx])))]
        b = boxes[idx]
        supp = np.zeros(len(idx), bool)
        nk = 0
        for i in range(len(idx)):
            if nk == max_per_class:
                break
            if supp[i]:
                continue
            nk += 1
            kept.append(int(idx[i]))
            js = np.arange(i + 1, len(idx))
            hit = iou_row(b, i, js) > threshold
            removed += int((hit & ~supp[js]).sum())
            supp[js[hit]] = True
    return np.array(kept, np.int64), removed


def detection_layer(rois: np.ndarray, logits: np.ndarray, deltas: np.ndarray, win: np.ndarray):
    """refine_detections_graph -> (count, detections [100, 6] y1 x1 y2 x2 class score zero padded, number removed by per-class NMS)"""
    n = rois.shape[0]
    cls, score = softmax_argmax(logits)
    d = deltas.reshape(n, NUM_CLASSES, 4)[np.arange(n), cls]
    boxes = apply_box_deltas_window(rois, d, win)
    with np.errstate(invalid="ignore"):
        cand = np.nonzero((cls > 0) & (score >= MIN_CONFIDENCE))[0]
    kept, removed = class_nms(boxes, score, cls, cand)
    kept = kept[np.lexsort((kept, _score_key(score[kept])))] if kept.size else kept
    kept = kept[:MAX_DET]
    out = np.zeros((MAX_DET, 6), np.float32)
    out[:kept.size, :4] = boxes[kept]
    out[:kept.size, 4] = cls[kept].astype(np.float32)
    out[:kept.size, 5] = score[kept]
    return int(kept.size), out, removed


def sigmoid(x):
    """R-SIGMOID: 1 / (1 + det_expf(-x))"""
    with np.errstate(over="ignore"):
        return (f32(1.0) / (f32(1.0) + det_expf(-np.asarray(x, np.float32)))).astype(np.float32)


def select_masks(mask_logits: np.ndarray, dets: np.ndarray) -> np.ndarray:
    """mask logits [100, 14, 14, 2, 2, 81] -> [100, 28, 28]: the detection's own class (padding rows: class 0), sigmoid"""
    cls = dets[:, 4].astype(np.int64)
    m = np.take_along_axis(mask_logits, cls[:, None, None, None, None, None], axis=5)[..., 0]
    m = m.transpose(0, 1, 3, 2, 4).reshape(MAX_DET, MASK, MASK)          # [d][y][dy][x][dx]
    return sigmoid(m)


def unmold(dets: np.ndarray, win: np.ndarray, W: int, H: int):
    """R-UNMOLD: N = first row with class 0; boxes (float32) shifted and scaled from the window to [0, 1] in float32; denorm_boxes in
    float64 (x (H-1, W-1), + (0, 0, 1, 1)), np.around (half to even), int32; rows with (y2-y1)*(x2-x1) <= 0 dropped.
    -> list of (detection row, y1, x1, y2, x2, class id, score)"""
    zero = np.nonzero(dets[:, 4] == 0)[0]
    N = int(zero[0]) if zero.size else dets.shape[0]
    wy1, wx1, wy2, wx2 = win.astype(np.float32)
    wh, ww = f32(wy2 - wy1), f32(wx2 - wx1)
    out = []
    for d in range(N):
        y1, x1, y2, x2 = dets[d, :4].astype(np.float32)
        nb = np.array([(y1 - wy1) / wh, (x1 - wx1) / ww, (y2 - wy1) / wh, (x2 - wx1) / ww], np.float32)
        b = np.around(nb.astype(np.float64) * np.array([H - 1, W - 1, H - 1, W - 1], np.float64) + np.array([0, 0, 1, 1], np.float64)).astype(np.int32)
        if (int(b[2]) - int(b[0])) * (int(b[3]) - int(b[1])) <= 0:
            continue
        out.append((d, int(b[0]), int(b[1]), int(b[2]), int(b[3]), int(dets[d, 4]), dets[d, 5]))
    return out


def resize_mask(m: np.ndarray, h: int, w: int) -> np.ndarray:
    """R-RESIZE: the 28x28 mask resized to h x w as skimage resize(order=1, mode='constant', anti_aliasing=False) = scipy.ndimage.zoom(order=1,
    mode='grid-constant', grid_mode=True): input coordinate (o + 0.5) * (28 / n) - 0.5 per axis in float64, bilinear with 0 outside the
    grid (x first, then y), rounded to float32"""
    def axis(n):
        c = (np.arange(n, dtype=np.float64) + 0.5) * (28.0 / n) - 0.5
        i0 = np.floor(c)
        return i0.astype(np.int64), c - i0
    iy, fy = axis(h)
    ix, fx = axis(w)
    mp = np.zeros((MASK + 2, MASK + 2), np.float64)
    mp[1:-1, 1:-1] = m.astype(np.float64)

    def at(yy, xx):
        yy = np.clip(yy + 1, 0, MASK + 1); xx = np.clip(xx + 1, 0, MASK + 1)
        return mp[yy[:, None], xx[None, :]]
    fxb, fyb = fx[None, :], fy[:, None]
    top = (1.0 - fxb) * at(iy, ix) + fxb * at(iy, ix + 1)
    bot = (1.0 - fxb) * at(iy + 1, ix) + fxb * at(iy + 1, ix + 1)
    return ((1.0 - fyb) * top + fyb * bot).astype(np.float32)


MEAN_PIXEL = (123.7, 116.8, 103.9)


def resize_channel(img: np.ndarray, h: int, w: int) -> np.ndarray:
    """R-MOLD step 1: one channel resized to h x w as scipy.ndimage.zoom(order=1, mode='grid-constant', grid_mode=True) computes it, in its
    own float64 arithmetic: per axis zoom = in / out, c = (o + 0.5) * zoom - 0.5, taps i0 = floor(c) and i0 + 1 (0 outside the image),
    w0 = 1 - (c - i0), w1 = 1 - w0; the value is the sum of (tap * wy) * wx over (y0, x0), (y0, x1), (y1, x0), (y1, x1), left to right"""
    H, W = img.shape

    def axis(n, m):
        c = (np.arange(n, dtype=np.float64) + 0.5) * (np.float64(m) / np.float64(n)) - 0.5
        i0 = np.floor(c)
        w0 = 1.0 - (c - i0)
        return i0.astype(np.int64), w0, 1.0 - w0
    iy, wy0, wy1 = axis(h, H)
    ix, wx0, wx1 = axis(w, W)
    mp = np.zeros((H + 2, W + 2), np.float64)
    mp[1:-1, 1:-1] = img

    def at(yy, xx):
        return mp[np.clip(yy + 1, 0, H + 1)[:, None], np.clip(xx + 1, 0, W + 1)[None, :]]
    Y0, Y1, X0, X1 = wy0[:, None], wy1[:, None], wx0[None, :], wx1[None, :]
    v = at(iy, ix) * Y0 * X0
    v = v + at(iy, ix + 1) * Y0 * X1
    v = v + at(iy + 1, ix) * Y1 * X0
    return v + at(iy + 1, ix + 1) * Y1 * X1


def bf16_bits(x: np.ndarray) -> np.ndarray:
    """float32 -> bfloat16 bit patterns, round to nearest even (finite values)"""
    u = np.ascontiguousarray(x, np.float32).view(np.uint32).astype(np.uint64)
    return ((u + 0x7FFF + ((u >> 16) & 1)) >> 16).astype(np.uint16)


def mold_input(rgb: np.ndarray, S: int):
    """R-MOLD: resize_image(mode='square') + mold_image on an H x W x >= 3 uint8 image -> (S x S x 3 bf16 bit patterns, the resized uint8
    letter box).  Resized per channel (resize_channel), truncated to uint8, placed at (offx, offy) of an S x S x 3 zero image,
    float32(u8) - MEAN_PIXEL in float64 rounded to float32, rounded once to bf16"""
    H, W = rgb.shape[:2]
    _, nw, nh, ox, oy = mold_geometry(S, W, H)
    box = np.stack([resize_channel(rgb[..., c].astype(np.float64), nh, nw) for c in range(3)], -1).astype(np.uint8)
    img = np.zeros((S, S, 3), np.uint8)
    img[oy:oy + nh, ox:ox + nw] = box
    return bf16_bits((img.astype(np.float32) - np.array(MEAN_PIXEL)).astype(np.float32)), box


MOLD_KINDS = ("random", "flat", "smooth")


def mold_test_image(kind: str, W: int, H: int, seed: int = 0) -> np.ndarray:
    """H x W x 4 uint8 test images for the mould: random (0 and 255 in every channel, alpha random too), flat, or smooth with ramps"""
    rng = np.random.default_rng(seed)
    if kind == "random":
        img = rng.integers(0, 256, (H, W, 4)).astype(np.uint8)
        img[0, 0], img[-1, -1], img[H // 2, 0], img[0, W // 2] = 0, 255, 255, 0
        return img
    if kind == "flat":
        img = np.empty((H, W, 4), np.uint8)
        img[...] = (200, 1, 255, 7)
        return img
    yy, xx = np.mgrid[0:H, 0:W].astype(np.float64)
    rgb = [127.5 + 127.5 * np.sin(xx / 37.0) * np.cos(yy / 23.0), 255.0 * xx / max(W - 1, 1), 255.0 * (1.0 - yy / max(H - 1, 1))]
    return np.stack([np.floor(np.clip(c, 0, 255)) for c in rgb] + [np.full((H, W), 255.0)], -1).astype(np.uint8)


def unmold_mask(m: np.ndarray, box, H: int, W: int) -> np.ndarray:
    """utils.unmold_mask: resize to the box, >= 0.5, placed at the box in an H x W bool image.  Boxes of the detection layer lie inside
    the image; a box outside it (only through crafted detections) is cut at the image edge, where numpy would wrap a negative index or
    fail on the shape, and a box inverted in both axes paints nothing, where skimage would fail"""
    y1, x1, y2, x2 = box
    full = np.zeros((H, W), bool)
    if y2 <= y1 or x2 <= x1:
        return full
    r = resize_mask(m, y2 - y1, x2 - x1) >= f32(0.5)
    cy1, cx1, cy2, cx2 = max(y1, 0), max(x1, 0), min(y2, H), min(x2, W)
    if cy1 < cy2 and cx1 < cx2:
        full[cy1:cy2, cx1:cx2] = r[cy1 - y1:cy2 - y1, cx1 - x1:cx2 - x1]
    return full


def export(cid: int, score, min_score: float, class_filter=(), special=(), ordinal=0):
    """generate_id_image's per-detection rule -> id (uint8) or None"""
    if class_filter and cid not in class_filter:
        return None
    if not (float(np.float32(score)) >= min_score):
        return None
    val = ordinal + 1
    if cid in special:
        val = special[cid]
    return val & 0xFF


def id_image(dets: np.ndarray, masks: np.ndarray, win: np.ndarray, W: int, H: int, min_score=0.55, class_filter=(), special=()):
    """unmold_detections + generate_id_image: later exported detections overwrite earlier ones -> (id image, class ids, rois)"""
    img = np.zeros((H, W), np.uint8)
    cls, rois = [], []
    for d, y1, x1, y2, x2, cid, score in unmold(dets, win, W, H):
        v = export(cid, score, min_score, class_filter, special, len(cls))
        if v is None:
            continue
        img[unmold_mask(masks[d], (y1, x1, y2, x2), H, W)] = v
        cls.append(cid); rois.append([y1, x1, y2, x2])
    return img, cls, rois


def unmolded_result(dets: np.ndarray, masks: np.ndarray, win: np.ndarray, W: int, H: int) -> dict:
    """model.detect's result dict (masks H x W x N uint8) for api.generate_id_image"""
    u = unmold(dets, win, W, H)
    full = np.zeros((H, W, len(u)), np.uint8)
    for k, (d, y1, x1, y2, x2, _, _) in enumerate(u):
        full[:, :, k] = unmold_mask(masks[d], (y1, x1, y2, x2), H, W)
    return {"masks": full, "scores": np.array([r[6] for r in u], np.float32), "class_ids": np.array([r[5] for r in u], np.int32),
            "rois": np.array([r[1:5] for r in u], np.int32).reshape(-1, 4)}
