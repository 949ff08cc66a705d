"""Crafted inputs at the decision edges of the segmentation tail (csrc/mf_seg.cu, MfSegmentation.cpp:221-522).

Each generator returns a Case: a frame size, the context settings the tail reads (new-model size window, mask close), one or more calls
(Steps: inverted edge map, raw depth, instance mask + classes, projected-ID image, model list) run in order on ONE context / oracle state,
and `claims`: which side of which decision each call lands on.  tests/test_cpu_seg_cases.py checks every claim on the oracle
(orc_mfseg_cpu) with the quantities recomputed from the inputs (scipy labelling, numpy float32 thresholds); tests/test_gpu_seg_edges.py
runs every case through MaskFusion.debugSegment and the oracle and compares them.  Pure numpy plus the oracle: no GPU.

Claims, as (step, claim) pairs, points as (y, x):
  ("ncomp", n)                   nComponents (background included)
  ("cc", )                       labels after edge removal == 4-connected labelling of the edge map (scipy), up to numbering
  ("area", p, a)                 the component of p in the edge map has a pixels
  ("same", p, q) / ("diff", p, q) / ("zero", p)    labels after edge removal
  ("fill", y, x0, n)             row y: labels x0 .. x0+n-1 equal the label at x0-1, label x0+n is 0
  ("seg", p, v)                  fullSegmentation at p
  ("new", has, cls)              hasNewLabel, newClassID
  ("step", p, q, below)          |depth[q] - depth[p]| (float32) < 0.008 (double) == below, with the float32 difference one ulp from
                                 the other side
  ("t", p, m, d)                 the mask-m overlap of p's component is (int)(0.65f * csize) + d
  ("newsize", m, which, d)       mask m's pixel count is (size_t)(rel * P) + d, rel = minRelSizeNew ("min") or maxRelSizeNew ("max")
  ("ovl", m, model, d)           mask m's overlap with the model's projection is 0.05f * maskPixels + d
  ("absorb", p, model, d)        pixels of p's component after edge removal projected as `model`: 0.6f * csize + d
"""
from __future__ import annotations

import ctypes as C
from dataclasses import dataclass, field

import numpy as np

from tests import oracle_lib as ol

f32 = np.float32
NAN = f32(np.nan)
DEFAULT_CFG = dict(minRelSizeNew=0.015, maxRelSizeNew=0.4, segMorphMaskRadius=2, segMorphMaskIterations=0)


@dataclass
class Step:
    edges: np.ndarray                       # H x W uint8, 255 = not an edge
    depth: np.ndarray                       # H x W float32
    mask: np.ndarray | None = None          # H x W uint8 (values < len(classIDs)); None: no masks
    classIDs: tuple = ()
    projected: np.ndarray | None = None     # H x W uint8 model ids; None: all 0
    modelIDs: tuple = (0,)
    modelClassIDs: tuple = (0,)
    nextModelID: int = 1
    allowNew: bool = False


@dataclass
class Case:
    name: str
    W: int
    H: int
    steps: list
    claims: list = field(default_factory=list)
    cfg: dict = field(default_factory=lambda: dict(DEFAULT_CFG))

    def inputs(self, s: Step):
        """a step's inputs in the form both sides take"""
        shape = (self.H, self.W)
        return dict(edgesInv=s.edges, depth=s.depth, mask=s.mask, classIDs=np.asarray(s.classIDs, np.int32),
                    projectedIDs=np.zeros(shape, np.uint8) if s.projected is None else s.projected,
                    modelIDs=np.asarray(s.modelIDs, np.uint8), modelClassIDs=np.asarray(s.modelClassIDs, np.int32),
                    nextModelID=int(s.nextModelID), allowNew=bool(s.allowNew))


@dataclass
class Out:
    seg: np.ndarray
    labels: np.ndarray
    hasNew: int
    newClass: int
    nComponents: int


def run_oracle(case: Case):
    """orc_mfseg_cpu on every step of a case with one state kept across them -> [Out]"""
    L = ol.lib()
    W, H = case.W, case.H
    st = ol.MfsegState()
    L.orc_mfseg_state_init(C.byref(st), W, H)
    outs = []
    try:
        for s in case.steps:
            a = case.inputs(s)
            edges = np.ascontiguousarray(a["edgesInv"], np.uint8).copy()
            depth = np.ascontiguousarray(a["depth"], np.float32)
            mask = np.zeros((H, W), np.uint8) if a["mask"] is None else np.ascontiguousarray(a["mask"], np.uint8)
            cls = a["classIDs"] if a["classIDs"].size else np.zeros(1, np.int32)
            proj = np.ascontiguousarray(a["projectedIDs"], np.uint8)
            ids, mcls = a["modelIDs"], a["modelClassIDs"]
            seg = np.zeros((H, W), np.uint8)
            lab = np.zeros((H, W), np.int32)
            i = ol.MfsegIn(W, H, edges.ctypes.data_as(ol.u8p), depth.ctypes.data_as(ol.f32p), mask.ctypes.data_as(ol.u8p),
                           int(a["classIDs"].size), cls.ctypes.data_as(C.POINTER(C.c_int32)), proj.ctypes.data_as(ol.u8p), int(ids.size),
                           ids.ctypes.data_as(ol.u8p), mcls.ctypes.data_as(C.POINTER(C.c_int32)), a["nextModelID"], int(a["allowNew"]),
                           case.cfg["minRelSizeNew"], case.cfg["maxRelSizeNew"], case.cfg["segMorphMaskRadius"],
                           case.cfg["segMorphMaskIterations"])
            o = ol.MfsegOut()
            o.fullSegmentation = seg.ctypes.data_as(ol.u8p)
            o.labels = lab.ctypes.data_as(C.POINTER(C.c_int32))
            L.orc_mfseg_cpu(C.byref(st), C.byref(i), C.byref(o))
            outs.append(Out(seg, lab, int(o.hasNewLabel), int(o.newClassID), int(o.nComponents)))
    finally:
        L.orc_mfseg_state_free(C.byref(st))
    return outs


# ---------------------------------------------------------------- helpers
def _nan(W, H):
    return np.full((H, W), NAN, np.float32)


def _rects(W, H, rects, value=255):
    """edge map: 255 inside each (y0, y1, x0, x1) rectangle (inclusive), 0 elsewhere"""
    e = np.zeros((H, W), np.uint8)
    for (y0, y1, x0, x1) in rects:
        e[y0:y1 + 1, x0:x1 + 1] = value
    return e


def _first_n(img, rect, n, value):
    """set the first n pixels (raster order) of rect (inclusive) to value"""
    y0, y1, x0, x1 = rect
    ys, xs = np.mgrid[y0:y1 + 1, x0:x1 + 1]
    ys, xs = ys.ravel()[:n], xs.ravel()[:n]
    img[ys, xs] = value


def _centre(r):
    return ((r[0] + r[1]) // 2, (r[2] + r[3]) // 2)


# ---------------------------------------------------------------- connected components (all-NaN depth: the sweeps change nothing)
CC_SIZES = [(640, 480), (644, 484), (36, 20), (28, 12)]


def checkerboard(W, H):
    yy, xx = np.mgrid[0:H, 0:W]
    return (((xx + yy) % 2 == 0) * 255).astype(np.uint8)


def spiral(W, H):
    """one-pixel-wide path spiralling over the whole frame, arms one background pixel apart: a single component"""
    R, Cn = (H + 1) // 2, (W + 1) // 2
    e = np.zeros((H, W), np.uint8)
    top, bot, left, right = 0, R - 1, 0, Cn - 1
    path = []
    while top <= bot and left <= right:
        path += [(top, c) for c in range(left, right + 1)]
        path += [(r, right) for r in range(top + 1, bot + 1)]
        if top < bot:
            path += [(bot, c) for c in range(right - 1, left - 1, -1)]
        if left < right:
            path += [(r, left) for r in range(bot - 1, top, -1)]
        top, bot, left, right = top + 1, bot - 1, left + 1, right - 1
    prev = None
    for (r, c) in path:
        e[2 * r, 2 * c] = 255
        if prev is not None:
            e[prev[0] + r, prev[1] + c] = 255            # the pixel between two consecutive cells
        prev = (r, c)
    return e


def comb(W, H):
    """teeth on the even columns from the top, joined only by the last row"""
    e = np.zeros((H, W), np.uint8)
    e[:H - 1, 0::2] = 255
    e[H - 1, :] = 255
    return e


def staircase(W, H):
    """diagonal runs: every pixel touches the next one at a corner only"""
    yy, xx = np.mgrid[0:H, 0:W]
    return (((xx - yy) % 6 == 0) * 255).astype(np.uint8)


def tile_touch(W, H):
    """two-pixel dominoes straddling every vertical (columns 32k-1 | 32k) and horizontal (rows 16k-1 | 16k) tile edge: joined only
    across the edge; next to each, a pair with one background pixel between (two components); a 2 x 2 block on every tile corner"""
    e = np.zeros((H, W), np.uint8)
    for xb in range(32, W, 32):
        for y in range(1, H - 1, 6):
            e[y, xb - 1:xb + 1] = 255
            if xb + 2 < W and xb - 3 >= 0:
                e[y + 2 if y + 2 < H else y, xb - 3] = 255
                e[y + 2 if y + 2 < H else y, xb + 1] = 255
    for yb in range(16, H, 16):
        for x in range(3, W - 1, 7):
            e[yb - 1:yb + 1, x] = 255
    for yb in range(16, H, 16):
        for xb in range(32, W, 32):
            e[yb - 1:yb + 1, xb - 1:xb + 1] = 255
    return e


def corners(W, H):
    e = np.zeros((H, W), np.uint8)
    e[0, 0] = e[0, W - 1] = e[H - 1, 0] = e[H - 1, W - 1] = 255
    return e


CC_PATTERNS = {"checkerboard": checkerboard, "spiral": spiral, "comb": comb, "staircase": staircase, "tile_touch": tile_touch,
               "all_fg": lambda W, H: np.full((H, W), 255, np.uint8), "all_bg": lambda W, H: np.zeros((H, W), np.uint8),
               "corners": corners}


def cc_cases():
    out = []
    for (W, H) in CC_SIZES:
        for name, fn in CC_PATTERNS.items():
            e = fn(W, H)
            claims = [(0, ("cc",))]
            n_fg = int((e > 0).sum())
            if name == "checkerboard":
                claims.append((0, ("ncomp", W * H // 2 + 1)))
            elif name in ("spiral", "comb", "all_fg"):
                claims.append((0, ("ncomp", 2)))
            elif name in ("staircase", "corners"):
                claims.append((0, ("ncomp", n_fg + 1)))
            elif name == "all_bg":
                claims.append((0, ("ncomp", 1)))
            elif name == "tile_touch" and W > 32:
                claims.append((0, ("same", (1, 31), (1, 32))))
                claims.append((0, ("diff", (3, 29), (3, 33))))
            out.append(Case(f"cc_{name}_{W}x{H}", W, H, [Step(e, _nan(W, H))], claims))
    return out


# ---------------------------------------------------------------- edge removal
def area_cases():
    """a component S of area 49 / 50 / 51 one edge column right of a large component B, all at one depth: S < 50 is eaten by B (one
    column per sweep), S > 50 fills the edge ring around itself; 50 does neither"""
    W, H = 64, 48
    out = []
    B = (2, 45, 2, 20)
    for a, (rows, cols) in {49: (7, 7), 50: (5, 10), 51: (3, 17)}.items():
        S = (10, 10 + rows - 1, 22, 22 + cols - 1)
        e = _rects(W, H, [B, S])
        d = np.full((H, W), f32(1.0), np.float32)
        claims = [(0, ("area", (10, 22), a)), (0, ("area", _centre(B), (B[1] - B[0] + 1) * (B[3] - B[2] + 1)))]
        right_ring = (11, S[3] + 1)
        if a < 50:
            claims += [(0, ("same", (12, 22), _centre(B))), (0, ("same", (12, 25), _centre(B))), (0, ("diff", (12, 26), _centre(B)))]
        if a == 50:
            claims += [(0, ("diff", (12, 22), _centre(B))), (0, ("zero", right_ring))]
        if a > 50:
            claims += [(0, ("same", right_ring, (10, 22))), (0, ("diff", (10, 22), _centre(B)))]
        out.append(Case(f"edge_area_{a}", W, H, [Step(e, d)], claims))
    return out


def _step_depths():
    """(name, d0, d1): float32 depths whose float32 difference sits one ulp either side of 0.008"""
    lo = np.nextafter(f32(0.008), f32(0))            # 0.008f is the first float32 above 0.008
    hi = f32(0.008)
    res = [("zero_below", f32(0), lo), ("zero_at_0.008f", f32(0), hi)]
    one = f32(1.0)
    k = int(np.floor(0.008 * 2 ** 23))                # depths near 1 m differ in steps of 2^-23
    res += [("1m_below", one, f32(1.0 + k * 2.0 ** -23)), ("1m_above", one, f32(1.0 + (k + 1) * 2.0 ** -23))]
    return res


def depth_step_cases():
    W, H = 40, 24
    out = []
    for name, d0, d1 in _step_depths():
        e = _rects(W, H, [(2, 21, 2, 15)])
        d = _nan(W, H)
        d[:, :16] = d0
        d[:, 16] = d1
        below = bool(abs(float(f32(d1) - f32(d0))) < 0.008)
        claims = [(0, ("step", (10, 15), (10, 16), below))]
        claims.append((0, ("same", (10, 16), (10, 10))) if below else (0, ("zero", (10, 16))))
        out.append(Case(f"edge_depth_step_{name}", W, H, [Step(e, d)], claims))
    return out


_OFFS = [(-1, -1), (-1, 0), (-1, 1), (0, -1), (0, 1), (1, -1), (1, 0), (1, 1)]


def order_cases():
    """an edge pixel whose only qualifying neighbours (same depth) are one pixel of component A and one of component B: the first of the
    two in the sweep's neighbour order wins.  Four layouts (A | B split by a vertical, horizontal and two diagonal edge lines) give every
    pair of positions that two different components can occupy (20 of the 28; the other 8 pairs are 4-adjacent)"""
    layouts = {
        "vertical": (40, 48, lambda y, x: np.sign(x - 20), [(4 + 5 * k, 20) for k in range(9)]),
        "horizontal": (48, 40, lambda y, x: np.sign(y - 20), [(20, 4 + 5 * k) for k in range(9)]),
        "diag_sum": (48, 48, lambda y, x: np.sign(x + y - 48), [(4 + 5 * k, 44 - 5 * k) for k in range(9)]),
        "diag_diff": (48, 48, lambda y, x: np.sign(x - y), [(4 + 5 * k, 4 + 5 * k) for k in range(9)]),
    }
    out = []
    for name, (W, H, side, centres) in layouts.items():
        yy, xx = np.mgrid[0:H, 0:W]
        s = side(yy, xx)
        e = ((s != 0) * 255).astype(np.uint8)
        d = np.full((H, W), f32(9.0), np.float32)
        claims = []
        (cy, cx) = centres[0]
        pa = [k for k, (oy, ox) in enumerate(_OFFS) if s[cy + oy, cx + ox] < 0]
        pb = [k for k, (oy, ox) in enumerate(_OFFS) if s[cy + oy, cx + ox] > 0]
        pairs = [(a, b) for a in pa for b in pb]
        assert len(pairs) == 9 and len(centres) == 9
        for (cy, cx), (a, b) in zip(centres, pairs):
            assert s[cy, cx] == 0
            pa_ = (cy + _OFFS[a][0], cx + _OFFS[a][1]); pb_ = (cy + _OFFS[b][0], cx + _OFFS[b][1])
            for p in ((cy, cx), pa_, pb_):
                d[p] = f32(1.0)
            claims.append((0, ("same", (cy, cx), pa_ if a < b else pb_)))
            claims.append((0, ("diff", (cy, cx), pb_ if a < b else pa_)))
        out.append(Case(f"edge_order_{name}", W, H, [Step(e, d)], claims))
    return out


def band_cases():
    """an 8-pixel edge band at one depth with a qualifying component on its left only: five Jacobi sweeps fill exactly five columns
    (an in-place raster sweep fills the band in one).  The border rows and columns stay as they are"""
    W, H = 40, 24
    e = _rects(W, H, [(0, H - 1, 1, 9), (0, H - 1, 18, W - 1)])
    d = np.full((H, W), f32(1.0), np.float32)
    d[:, 18:] = f32(5.0)                               # right side: a component, but too far in depth
    claims = [(0, ("fill", y, 10, 5)) for y in (1, 10, H - 2)]
    claims += [(0, ("zero", (0, 12))), (0, ("zero", (H - 1, 12))), (0, ("zero", (10, 0)))]
    cases = [Case("edge_band_8px", W, H, [Step(e, d)], claims)]
    # zero depth is a depth like any other; NaN never qualifies
    e = _rects(W, H, [(2, 10, 2, 15), (13, 21, 2, 15)])
    d = np.full((H, W), f32(0.0), np.float32)
    d[12:, :] = NAN
    cases.append(Case("edge_zero_and_nan_depth", W, H, [Step(e, d)],
                      [(0, ("same", (5, 16), (5, 10))), (0, ("zero", (17, 16))), (0, ("zero", (5, W - 1)))]))
    return cases


# ---------------------------------------------------------------- mask mapping and vote (160 x 120: minNew 288, maxNew 7680)
VW, VH = 160, 120


def _vote_case(name, rects, masks, classIDs, proj=None, models=((0, 0),), nextID=20, allowNew=True, claims=(), cfg=None, W=VW, H=VH):
    """rects: components; masks: [(mask id, rect, n or None)] -> mask id on the first n pixels (all if None); proj: [(model id, rect, n)]"""
    e = _rects(W, H, rects)
    m = np.zeros((H, W), np.uint8)
    for (mid, r, n) in masks:
        _first_n(m, r, (r[1] - r[0] + 1) * (r[3] - r[2] + 1) if n is None else n, mid)
    p = np.zeros((H, W), np.uint8)
    for (pid, r, n) in proj or ():
        _first_n(p, r, (r[1] - r[0] + 1) * (r[3] - r[2] + 1) if n is None else n, pid)
    c = dict(DEFAULT_CFG, **(cfg or {}))
    st = Step(e, _nan(W, H), m, tuple(classIDs), p, tuple(i for i, _ in models), tuple(k for _, k in models), nextID, allowNew)
    return Case(name, W, H, [st], [(0, cl) for cl in claims], c)


def vote_cases():
    out = []
    small = {"minRelSizeNew": 0.005}                   # minNew 96: a single mapped component of 161 pixels can become a model
    r160, r161 = (10, 19, 10, 25), (10, 16, 30, 52)    # 10 x 16, 7 x 23
    for r, a in ((r160, 160), (r161, 161)):
        out.append(_vote_case(f"vote_csize_{a}", [r], [(1, r, None)], [0, 4], claims=[
            ("area", _centre(r), a), ("seg", _centre(r), 0 if a == 160 else 20), ("new", int(a > 160), 4 if a > 160 else -1)], cfg=small))
    r400 = (10, 29, 10, 29)
    t = int(f32(0.65) * f32(400))                      # 260 in float32 (259 in double)
    for dlt in (0, 1):
        out.append(_vote_case(f"vote_overlap_t{'+1' if dlt else ''}", [r400], [(1, r400, t + dlt)], [0, 4], claims=[
            ("t", (20, 20), 1, dlt), ("seg", (20, 20), 20 if dlt else 0), ("new", dlt, 4 if dlt else -1)]))
    ra, rb = (10, 19, 10, 29), (30, 39, 10, 29)        # 200 + 200: only their sum passes minNew
    out.append(_vote_case("vote_mask_of_two_components", [ra, rb], [(1, ra, None), (1, rb, None)], [0, 6], claims=[
        ("area", _centre(ra), 200), ("area", _centre(rb), 200), ("newsize", 1, "min", 112), ("seg", _centre(ra), 20),
        ("seg", _centre(rb), 20), ("new", 1, 6)]))
    models = ((0, 0), (7, 3))
    for ov in (19, 20):                                # 0.05f * 400 = 20
        out.append(_vote_case(f"vote_model_overlap_{ov}", [r400], [(1, r400, None)], [0, 3], proj=[(7, r400, ov)], models=models, claims=[
            ("ovl", 1, 7, ov - 20), ("seg", (25, 25), 20 if ov < 20 else 7), ("new", int(ov < 20), 3 if ov < 20 else -1)]))
    for cls, want in ((3, 7), (4, 255)):
        out.append(_vote_case(f"vote_class_{'match' if cls == 3 else 'mismatch'}", [r400], [(1, r400, None)], [0, cls],
                              proj=[(7, r400, 200)], models=models, claims=[("seg", (25, 25), want), ("new", 0, -1)]))
    # the new-model size window, strict on both ends
    for which, size, rect in (("min", 0, (10, 25, 10, 27)), ("min", 1, (10, 26, 10, 26)),      # 288, 289
                              ("max", 0, (10, 89, 10, 105)), ("max", -1, (10, 89, 10, 105))):  # 7680, 7680 - 1
        e_rect = [rect]
        masks = [(1, rect, None)]
        case = _vote_case(f"vote_new_{which}{'%+d' % size if size else ''}", e_rect, masks, [0, 5], claims=[
            ("newsize", 1, which, size), ("new", int(size != 0), 5 if size else -1), ("seg", _centre(rect), 20 if size else 255)])
        if which == "max" and size == -1:
            case.steps[0].edges[10, 10] = 0             # one pixel less
            case.steps[0].mask[10, 10] = 0
        out.append(case)
    # two masks that could both become a model: the first one wins; none with allowNew = 0
    r1, r2 = (10, 29, 10, 29), (40, 59, 10, 29)
    for allow in (True, False):
        out.append(_vote_case(f"vote_two_new_allow{int(allow)}", [r1, r2], [(1, r1, None), (2, r2, None)], [0, 8, 9], allowNew=allow,
                              claims=[("seg", _centre(r1), 20 if allow else 255), ("seg", _centre(r2), 255),
                                      ("new", int(allow), 8 if allow else -1)]))
    out.append(_many_case())
    return out


def _many_case():
    """256 masks (mask ids 1..255 on their own 13 x 13 component) and 63 models (ids 0..62); mask k overlaps model 1 + k % 62 on 100
    pixels, with its class on two masks of three; masks 7 and 8 overlap no model: 7 becomes the new model, 8 is dropped"""
    W, H = 320, 240
    rects = []
    for gy in range(H // 14):
        for gx in range(W // 14):
            rects.append((gy * 14 + 1, gy * 14 + 13, gx * 14 + 1, gx * 14 + 13))
    rects = rects[:255]
    models = [(j, j % 5) for j in range(63)]
    masks, proj, cls, claims = [], [], [0], []
    for k in range(1, 256):
        r = rects[k - 1]
        j = 1 + k % 62
        masks.append((k, r, None))
        cls.append(j % 5 if k % 3 else (j % 5) + 1)
        if k in (7, 8):
            want = 63 if k == 7 else 255
        else:
            proj.append((j, r, 100))
            want = j if k % 3 else 255
        if k < 255:
            claims.append(("seg", _centre(r), want))
    claims.append(("new", 1, cls[7]))
    return _vote_case("vote_256_masks_63_models", rects, masks, cls, proj=proj, models=models, nextID=63, claims=claims, W=W, H=H,
                      cfg={"minRelSizeNew": 0.001})      # minNew 76: a 169-pixel mask can become a model


# ---------------------------------------------------------------- absorb of the components no mask took (96 x 64, models 0, 7, 9)
AW, AH = 96, 64
AMODELS = ((0, 0), (7, 1), (9, 2))


def _absorb_case(name, e, d, p, claims):
    st = Step(e, d, None, (), p, tuple(i for i, _ in AMODELS), tuple(k for _, k in AMODELS), 20, False)
    return Case(name, AW, AH, [st], [(0, c) for c in claims])


def absorb_cases():
    out = []
    # tie: a 10 x 10 component grows to 20 x 20 in the sweeps; its pixels then split 200 / 200 between models 7 and 9: the first wins
    e = _rects(AW, AH, [(20, 29, 20, 29)])
    d = _nan(AW, AH); d[15:35, 15:35] = f32(1.0)
    p = np.zeros((AH, AW), np.uint8); p[15:35, 15:25] = 7; p[15:35, 25:35] = 9
    out.append(_absorb_case("absorb_tie_first_model", e, d, p, [("absorb", (25, 25), 7, 200 - 60), ("absorb", (25, 25), 9, 200 - 60),
                                                                ("seg", (25, 25), 7), ("seg", (22, 28), 7)]))
    # exactly 0.6f * csize (= 180 of 300) and one more
    r = (20, 34, 20, 39)
    for dlt in (0, 1):
        p = np.zeros((AH, AW), np.uint8); _first_n(p, r, 180 + dlt, 7)
        out.append(_absorb_case(f"absorb_overlap_0.6{'+1' if dlt else ''}", _rects(AW, AH, [r]), _nan(AW, AH), p,
                                [("absorb", (27, 30), 7, dlt), ("seg", (27, 30), 7 if dlt else 0)]))
    # the background wins the max: 210 pixels projected 0, 190 projected 7 (> 0.6f * 100) after the sweeps
    e = _rects(AW, AH, [(20, 29, 20, 29)])
    d = _nan(AW, AH); d[15:35, 15:35] = f32(1.0)
    p = np.zeros((AH, AW), np.uint8); _first_n(p, (15, 34, 15, 34), 190, 7)
    out.append(_absorb_case("absorb_background_wins", e, d, p, [("absorb", (25, 25), 7, 190 - 60), ("seg", (25, 25), 0)]))
    # the box rule: pixels the sweeps added are absorbed up to right + 1 / bottom + 1 of the pre-sweep box, not beyond, not left / above
    e = _rects(AW, AH, [(20, 39, 20, 39)])
    d = _nan(AW, AH); d[10:50, 10:50] = f32(1.0)
    p = np.zeros((AH, AW), np.uint8); p[10:50, 10:50] = 7
    out.append(_absorb_case("absorb_box_plus_one", e, d, p, [
        ("seg", (30, 30), 7), ("seg", (30, 40), 7), ("seg", (40, 30), 7), ("seg", (40, 40), 7), ("seg", (30, 41), 0), ("seg", (41, 30), 0),
        ("seg", (30, 19), 0), ("seg", (19, 30), 0), ("same", (30, 41), (30, 30)), ("same", (19, 30), (30, 30))]))
    # components on the right and the bottom border
    rr, rb = (20, 39, 70, AW - 1), (50, AH - 1, 10, 30)
    p = np.zeros((AH, AW), np.uint8); p[20:40, 70:] = 7; p[50:, 10:31] = 9
    out.append(_absorb_case("absorb_at_right_and_bottom_border", _rects(AW, AH, [rr, rb]), _nan(AW, AH), p,
                            [("seg", (30, AW - 1), 7), ("seg", (AH - 1, 20), 9), ("seg", (AH - 1, 30), 9)]))
    return out


# ---------------------------------------------------------------- state that persists across calls (ignore map, maskToID)
def persistent_cases():
    W, H = VW, VH
    cfg = dict(DEFAULT_CFG, segMorphMaskIterations=1)   # the mask close runs (radius 2) whenever the call has masks
    c1, c2, c3, c5, c6 = (10, 39, 10, 49), (10, 39, 60, 99), (50, 89, 10, 49), (10, 39, 110, 149), (95, 115, 110, 149)
    c4 = (55, 85, 65, 105)
    persons = [(60, 79, 70, 84), (60, 79, 87, 100)]     # two person boxes two pixels apart: the close fills the gap
    e = _rects(W, H, [c1, c2, c3, c4, c5, c6])
    d = _nan(W, H)
    proj = np.zeros((H, W), np.uint8); proj[c1[0]:c1[1] + 1, c1[2]:c1[3] + 1] = 7
    models = dict(modelIDs=(0, 7), modelClassIDs=(0, 3), nextModelID=8, allowNew=True)

    def masks(spec):
        m = np.zeros((H, W), np.uint8)
        for k, r in spec:
            m[r[0]:r[1] + 1, r[2]:r[3] + 1] = k
        return m
    person = masks([(1, c1), (2, persons[0]), (2, persons[1])])
    steps = [Step(e, d, person, (0, 3, 255), proj, **models),          # person: ignored, its edges removed
             Step(e, d, None, (), proj, **models),                       # no masks: the ignore map stays, the close does not run
             Step(e, d, masks([(1, c1)]), (0, 3), proj, **models),       # masks without a person: the ignore map is cleared
             Step(e, d, masks([(1, c1), (2, c2), (3, c3), (4, c5), (5, c6)]), (0, 3, 1, 2, 4, 5), proj, **models),   # 6 masks
             Step(e, d, masks([(1, c2), (2, c3)]), (0, 2, 1), proj, **models)]                                       # then 3
    claims = [(0, ("seg", (70, 75), 255)), (0, ("seg", (70, 85), 255)), (0, ("seg", _centre(c1), 7)),
              (1, ("seg", (70, 75), 255)), (1, ("seg", (70, 85), 0)), (1, ("zero", (70, 75))), (1, ("seg", _centre(c1), 7)),
              (2, ("seg", (70, 75), 0)), (2, ("same", (70, 75), (57, 67))),
              (3, ("seg", _centre(c1), 7)), (3, ("seg", _centre(c2), 8)), (3, ("seg", _centre(c3), 255)), (3, ("new", 1, 1)),
              (4, ("seg", _centre(c2), 8)), (4, ("seg", _centre(c3), 255)), (4, ("new", 1, 2))]
    return [Case("state_ignore_map_and_mask_ids", W, H, steps, claims, cfg)]


def all_cases():
    return cc_cases() + area_cases() + depth_step_cases() + order_cases() + band_cases() + vote_cases() + absorb_cases() + persistent_cases()
