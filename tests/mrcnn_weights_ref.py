"""numpy restatement of the pretrained-weight path (csrc/mf_weights.cu, DESIGN §3c): matterport's Keras layer names and kernel shapes,
seeded stand-in weights in the Keras layouts, and R-FOLD + relayout into the handles' [rows x K] tables.  Written from the architecture
description, not from the C++ tables, so that the two pin each other."""
from __future__ import annotations

import numpy as np

from tests.rpn_ref import to_bf16_bits

f32, f64 = np.float32, np.float64
EPS = 1e-3                                     # Keras BatchNormalization default, matterport's BatchNorm keeps it


def _ceil64(k):
    return (k + 63) // 64 * 64


def backbone_layers():
    """[(conv layer, BatchNorm layer or None, Keras kernel shape)] in the backbone's layer-table order (mf_backbone_create): conv1, per block
    branch2a / 2b / 2c and (block a) branch1, fpn_c2p2..c5p5, fpn_p2..p5"""
    out = [("conv1", "bn_conv1", (7, 7, 3, 64))]
    cin = 64
    for st, nb, f in ((2, 3, 64), (3, 4, 128), (4, 23, 256), (5, 3, 512)):
        for blk in range(nb):
            b = chr(ord("a") + blk)                  # stage 4 of ResNet-101: a, then b..w
            out += [(f"res{st}{b}_branch2a", f"bn{st}{b}_branch2a", (1, 1, cin, f)),
                    (f"res{st}{b}_branch2b", f"bn{st}{b}_branch2b", (3, 3, f, f)),
                    (f"res{st}{b}_branch2c", f"bn{st}{b}_branch2c", (1, 1, f, 4 * f))]
            if blk == 0:
                out.append((f"res{st}a_branch1", f"bn{st}a_branch1", (1, 1, cin, 4 * f)))
            cin = 4 * f
    out += [(f"fpn_c{l}p{l}", None, (1, 1, c, 256)) for l, c in ((2, 256), (3, 512), (4, 1024), (5, 2048))]
    out += [(f"fpn_p{l}", None, (3, 3, 256, 256)) for l in (2, 3, 4, 5)]
    return out


RPN_LAYERS = [("rpn_conv_shared", None, (3, 3, 256, 512)), ("rpn_class_raw", None, (1, 1, 512, 6)), ("rpn_bbox_pred", None, (1, 1, 512, 12))]
DETECTOR_LAYERS = ([("mrcnn_class_conv1", "mrcnn_class_bn1", (7, 7, 256, 1024)), ("mrcnn_class_conv2", "mrcnn_class_bn2", (1, 1, 1024, 1024)),
                    ("mrcnn_class_logits", None, (1024, 81)), ("mrcnn_bbox_fc", None, (1024, 324))] +
                   [(f"mrcnn_mask_conv{i}", f"mrcnn_mask_bn{i}", (3, 3, 256, 256)) for i in (1, 2, 3, 4)] +
                   [("mrcnn_mask_deconv", None, (2, 2, 256, 256)), ("mrcnn_mask", None, (1, 1, 256, 81))])
ALL_LAYERS = {"backbone": backbone_layers(), "rpn": RPN_LAYERS, "detector": DETECTOR_LAYERS}


def handle_tables():
    """{part: [(handle layer name, [Keras layers], rows, K)]} in each handle's table order"""
    bb = [(n, [n], s[3], _ceil64(s[0] * s[1] * s[2])) for n, _, s in backbone_layers()]
    rpn = [("rpn_conv_shared", ["rpn_conv_shared"], 512, 2304), ("rpn_class_raw+rpn_bbox_pred", ["rpn_class_raw", "rpn_bbox_pred"], 64, 512)]
    det = [("mrcnn_class_conv1", ["mrcnn_class_conv1"], 1024, 12544), ("mrcnn_class_conv2", ["mrcnn_class_conv2"], 1024, 1024),
           ("mrcnn_class_logits+mrcnn_bbox_fc", ["mrcnn_class_logits", "mrcnn_bbox_fc"], 448, 1024)]
    det += [(f"mrcnn_mask_conv{i}", [f"mrcnn_mask_conv{i}"], 256, 2304) for i in (1, 2, 3, 4)]
    det += [("mrcnn_mask_deconv", ["mrcnn_mask_deconv"], 1024, 256), ("mrcnn_mask", ["mrcnn_mask"], 128, 256)]
    return {"backbone": bb, "rpn": rpn, "detector": det}


def _bn_of():
    return {n: bn for layers in ALL_LAYERS.values() for n, bn, _ in layers}


def _shape_of():
    return {n: s for layers in ALL_LAYERS.values() for n, _, s in layers}


def make_weights(seed: int, parts=("backbone", "rpn", "detector")) -> dict:
    """seeded stand-in weights {"<layer>/<param>": float32 array} in the Keras layouts: He-scaled kernels, small biases, BatchNorm statistics
    that keep activations O(1) (moving_variance in [0.5, 2], small moving_mean, gamma < 1 on branch2c so residual sums stay bounded).  The
    moulded input is in pixel units (std ~ 60), so bn_conv1's variance is that of the stem's output, ~1e4: the stem then normalises it."""
    rng = np.random.default_rng(seed)
    out = {}
    for part in parts:
        for name, bn, shape in ALL_LAYERS[part]:
            fan_in = shape[3] if name == "mrcnn_mask_deconv" else int(np.prod(shape[:-1]))
            cout = shape[2] if name == "mrcnn_mask_deconv" else shape[-1]
            out[f"{name}/kernel"] = (rng.standard_normal(shape) * np.sqrt(2.0 / fan_in)).astype(f32)
            out[f"{name}/bias"] = (rng.standard_normal(cout) * 0.05).astype(f32)
            if bn:
                lo, hi = (0.2, 0.5) if name.endswith("branch2c") else (0.7, 1.2)
                out[f"{bn}/gamma"] = rng.uniform(lo, hi, cout).astype(f32)
                out[f"{bn}/beta"] = (rng.standard_normal(cout) * 0.05).astype(f32)
                out[f"{bn}/moving_mean"] = (rng.standard_normal(cout) * 0.1).astype(f32)
                out[f"{bn}/moving_variance"] = (rng.uniform(0.5, 2.0, cout) * (1e4 if name == "conv1" else 1.0)).astype(f32)
    return out


def bf16(x) -> np.ndarray:
    return (to_bf16_bits(x).astype(np.uint32) << 16).view(f32)


def fold(t: dict, name: str):
    """R-FOLD of Keras layer `name`: -> (bf16-rounded kernel in its Keras layout, float32 bias [cout])"""
    k, b = t[f"{name}/kernel"], t[f"{name}/bias"]
    bn = _bn_of()[name]
    if bn is None:
        return bf16(k), b.astype(f32)
    s = t[f"{bn}/gamma"].astype(f64) / np.sqrt(t[f"{bn}/moving_variance"].astype(f64) + EPS)
    shift = (b.astype(f64) - t[f"{bn}/moving_mean"].astype(f64)) * s + t[f"{bn}/beta"].astype(f64)
    return bf16((k.astype(f64) * s).astype(f32)), shift.astype(f32)


def table(t: dict, handle_layer: str):
    """the handle's [rows x K] weights and [rows] bias of `handle_layer`, folded and relaid out, zero padded"""
    spec = {n: (parts, rows, K) for tabs in handle_tables().values() for n, parts, rows, K in tabs}
    parts, rows, K = spec[handle_layer]
    W = np.zeros((rows, K), f32); B = np.zeros(rows, f32)
    r0 = 0
    for name in parts:
        w, b = fold(t, name)
        if name == "mrcnn_mask_deconv":            # (dy, dx, out, in) -> row (dy*2 + dx)*out + o, column c; the bias per (dy, dx) block
            W[:4 * w.shape[2], :w.shape[3]] = w.reshape(4 * w.shape[2], w.shape[3])
            B[:4 * w.shape[2]] = np.tile(b, 4)
            continue
        if w.ndim == 2:                            # Dense (in, out) -> row o, column i
            W[r0:r0 + w.shape[1], :w.shape[0]] = w.T
        else:                                      # Conv2D (kh, kw, cin, cout) -> row o, column (ky*kw + kx)*cin + c
            W[r0:r0 + w.shape[3], :w[..., 0].size] = w.transpose(3, 0, 1, 2).reshape(w.shape[3], -1)
        B[r0:r0 + b.size] = b
        r0 += b.size
    return W, B
