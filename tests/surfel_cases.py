"""Crafted surfel stores at the decision edges of the index map, clean and splat passes (csrc/mf_surfel.cu).

Each generator returns a Case: a store (N x 12 float32, the layout of Model::downloadMap), a pose, a depth / rgb frame, the config
overrides and a `claims` dict that says which edges the store hits.  Edges are found by search in float32, not hoped for: with
-fmad=false on mf_surfel.cu and -ffp-contract=off in the oracle, x = ((fx * X) / Z) + cx evaluated on numpy float32 scalars is the
kernels' arithmetic, and under the identity pose the transform is exact.  Sprite size and range come from the oracle itself
(orc_splat_extent).  Pure numpy plus the oracle: no GPU.  tests/test_cpu_surfel_cases.py checks every claim; tests/test_gpu_surfel_edges.py
runs every case through the CUDA passes and the oracle and compares them bit for bit.
"""
from __future__ import annotations

import ctypes as C
import functools
from dataclasses import dataclass, field

import numpy as np

from tests import oracle_lib as ol

W, H = 640, 480
f32 = np.float32
FX, FY, CX, CY = f32(528.0), f32(528.0), f32(320.0), f32(240.0)     # default camera at 640x480
MAXD = f32(20.0)             # maxDepthProcessed: depth range of the index map and the splat
CONF = f32(10.0)             # confGlobal: the background model's confidence threshold
TICK = 30                    # frame time of every case; the splat's maxTime is the same
PLANE_Z = 3.5                # depth of the plane frame (inside depthCutoff = 4)
NEW_ON_PLANE = (W // 2) * (H // 2)   # pixels the association emits a new vertex for on the plane (x, y of TICK's parity, P / 4)
BIG_N = 1_100_000
IDENT = np.eye(4, dtype=np.float32)


@dataclass
class Case:
    name: str
    kind: str                    # "index", "clean", "splat" or "time"
    store: np.ndarray
    pose: np.ndarray
    depth: np.ndarray
    rgb: np.ndarray
    cfg: dict
    claims: dict
    survivors: int | None = None     # clean cases: the oracle's designed store count after Model::clean
    removed: np.ndarray | None = field(default=None, repr=False)


def nxt(v, d=np.inf):
    return np.nextafter(f32(v), f32(d), dtype=np.float32)


def proj(X, Z, f, c):
    """the kernels' projection of one coordinate, in float32: ((f * X) / Z) + c"""
    return f32(f32(f32(f) * f32(X)) / f32(Z)) + f32(c)


def solve(target, Z, f, c, steps=512):
    """float32 X with proj(X, Z, f, c) == target exactly, or None"""
    target, Z = f32(target), f32(Z)
    X = f32((float(target) - float(c)) * float(Z) / float(f))
    for _ in range(steps):
        x = proj(X, Z, f, c)
        if x == target:
            return X
        X = nxt(X, np.inf if x < target else -np.inf)
    return None


def solve_any(target, f, c):
    for k in range(400):
        Z = f32(2.0625 + k / 97.0)
        X = solve(target, Z, f, c, steps=64)
        if X is not None:
            return X, f32(Z)
    raise AssertionError(f"no float32 position projects exactly onto {target!r}")


def solve_below(target, f, c):
    """the position whose projection is the largest float32 value below `target` that the projection can produce (for x near 100
    the step is ulp(x - cx), coarser than ulp(x))"""
    X, Z = solve_any(target, f, c)
    while proj(X, Z, f, c) >= f32(target):
        X = nxt(X, -np.inf)
    return X, Z


def surfel(x, y, z, conf=20.0, init=1.0, last=TICK, n=(0.0, 0.0, -1.0), rad=0.002, color=0x336699):
    return np.array([x, y, z, conf, float(color), 0.0, init, last, n[0], n[1], n[2], rad], np.float32)


def frame(kind):
    rgb = np.zeros((H, W, 3), np.uint8)
    rgb[..., 0] = (np.arange(W) % 251)[None, :]; rgb[..., 1] = (np.arange(H) % 241)[:, None]; rgb[..., 2] = 97
    depth = np.zeros((H, W), np.float32) if kind == "zero" else np.full((H, W), PLANE_Z, np.float32)
    return np.ascontiguousarray(depth), rgb


def rotated_pose(seed=3):
    """camera-to-world pose: a small rotation and a translation (the general, inexact transform)"""
    rng = np.random.default_rng(seed)
    w = rng.normal(size=3); w *= 0.12 / np.linalg.norm(w)
    th = np.linalg.norm(w); k = w / th
    K = np.array([[0, -k[2], k[1]], [k[2], 0, -k[0]], [-k[1], k[0], 0]])
    T = np.eye(4)
    T[:3, :3] = np.eye(3) + np.sin(th) * K + (1 - np.cos(th)) * K @ K
    T[:3, 3] = rng.normal(size=3) * 0.3
    return T.astype(np.float32)


def to_world(pose, cam_pts, cam_nrm):
    """camera-space points / normals -> world (float64, rounded once)"""
    T = pose.astype(np.float64)
    return ((cam_pts @ T[:3, :3].T) + T[:3, 3]).astype(np.float32), (cam_nrm @ T[:3, :3].T).astype(np.float32)


# ---- the oracle's sprite of one surfel (splat.vert + R-PR), so that no third restatement of size and range exists ----
def _lib():
    L = ol.lib()
    if not getattr(L.orc_splat_extent, "_bound", False):
        L.orc_splat_extent.restype = None
        L.orc_splat_extent.argtypes = [C.c_void_p, C.c_void_p, ol.Cam, C.c_int, C.c_int, C.c_float, C.c_float, C.c_int, C.c_int,
                                       C.c_int, C.c_void_p]
        L.orc_splat_extent._bound = True
    return L


@dataclass
class Sprite:
    ok: bool; size: float; xw: float; yw: float; x0: int; x1: int; y0: int; y1: int
    pos: np.ndarray; n: np.ndarray; rad: float


def splat_extent(s, pose=IDENT, conf=CONF, time=TICK, max_time=TICK, time_delta=2**30 - 1):
    s = np.ascontiguousarray(s, np.float32); pose = np.ascontiguousarray(pose, np.float32); o = np.zeros(16, np.float32)
    _lib().orc_splat_extent(ol.ptr(s), ol.ptr(pose), ol.cam(FX, FY, CX, CY), W, H, C.c_float(MAXD), C.c_float(conf), time, max_time,
                            time_delta, ol.ptr(o))
    return Sprite(bool(o[0]), o[1], o[2], o[3], int(o[4]), int(o[5]), int(o[6]), int(o[7]), o[8:11].copy(), o[11:14].copy(), o[14])


def dot3(a, b):
    return f32(f32(f32(a[0] * b[0]) + f32(a[1] * b[1])) + f32(a[2] * b[2]))


def pixel_ray(px, py):
    """combo_splat.frag's viewing ray of pixel (px, py), float32 (R-NORM)"""
    l = [f32(f32(f32(px) + f32(0.5)) - CX) / FX, f32(f32(f32(py) + f32(0.5)) - CY) / FY, f32(1.0)]
    n = np.sqrt(dot3(l, l), dtype=np.float32)
    return [f32(l[0] / n), f32(l[1] / n), f32(l[2] / n)]


def disc_dd(sp: Sprite, px, py):
    """(dot(d, d), rad * rad) of the disc test of combo_splat.frag at one pixel, float32"""
    l = pixel_ray(px, py)
    t = f32(dot3(sp.pos, sp.n) / dot3(l, sp.n))
    d = [f32(f32(t * l[k]) - sp.pos[k]) for k in range(3)]
    return dot3(d, d), f32(f32(sp.rad) * f32(sp.rad))


# ======================================================================================================================================
# index map: k_index_project / k_index_resolve and the copy of the projection in k_clean_p1
# ======================================================================================================================================
def index_edges():
    rows, claims = [], {}

    def add(key, s, k=1):
        rows.append(s); claims[key] = claims.get(key, 0) + k

    # ties at equal zn on one pixel; the first group holds store index 0 (N2: id 0 is "no surfel" to the readers of the index map)
    groups = []
    for gi, (n, order) in enumerate([(3, 1), (2, -1), (17, 1), (17, -1), (64, 1), (64, -1), (2, 1), (5, -1)]):
        px, py = 40 + 70 * gi, 60 + 7 * gi
        Z = f32(1.5)
        xs = [f32((px + 0.1 + 0.8 * j / n - float(CX)) * float(Z) / float(FX)) for j in range(n)][::order]
        Y = f32((py + 0.5 - float(CY)) * float(Z) / float(FY))
        groups.append(len(rows))
        for X in xs:
            rows.append(surfel(X, Y, Z))
    claims["tie_groups"] = 8; claims["tie_group_with_id0"] = 1; claims["tie_max"] = 64
    # hundreds on one pixel at distinct depths (shuffled)
    rng = np.random.default_rng(11)
    zs = np.linspace(1.0, 3.0, 300).astype(np.float32)[rng.permutation(300)]
    for Z in zs:
        X = f32((500.4 - float(CX)) * float(Z) / float(FX)); Y = f32((300.6 - float(CY)) * float(Z) / float(FY))
        rows.append(surfel(X, Y, Z))
    claims["stack_distinct_depths"] = 300
    # x exactly at integers, one step below (negative target: the largest projection below it), 0, W - ulp, W (each on a row of its own)
    r = 380
    for tgt, key in [(100, "x_integer"), (321, "x_integer"), (-100, "x_ulp_below_integer"), (-321, "x_ulp_below_integer"),
                     (0, "x_zero"), (-W, "x_W_minus_ulp"), (W, "x_W")]:
        X, Z = solve_below(-tgt, FX, CX) if tgt < 0 else solve_any(tgt, FX, CX)
        add(key, surfel(X, f32((r + 0.5 - float(CY)) * float(Z) / float(FY)), Z)); r += 5
    c = 550
    for tgt, key in [(200, "y_integer"), (-200, "y_ulp_below_integer"), (0, "y_zero"), (-H, "y_H_minus_ulp"), (H, "y_H")]:
        Y, Z = solve_below(-tgt, FY, CY) if tgt < 0 else solve_any(tgt, FY, CY)
        add(key, surfel(f32((c + 0.5 - float(CX)) * float(Z) / float(FX)), Y, Z)); c += 5
    # depth: Z == maxDepthProcessed (zn == 1: not drawn), one ulp below (zn < 1), one ulp above, 0 and -0
    for Z, key in [(MAXD, "z_maxdepth"), (nxt(MAXD, 0), "z_maxdepth_minus_ulp"), (nxt(MAXD), "z_maxdepth_plus_ulp"),
                   (f32(0.0), "z_zero"), (f32(-0.0), "z_negzero")]:
        add(key, surfel(f32(0.25), f32(-0.5), Z, rad=0.05))
    store = np.stack(rows)
    depth, rgb = frame("zero")
    return Case("index_edges", "index", store, IDENT, depth, rgb, {}, claims)


def index_general():
    """a rotated pose over surfels in front of the camera, with repeated positions (ties under an inexact transform)"""
    rng = np.random.default_rng(5)
    n = 4000
    pc = np.stack([rng.uniform(-1.2, 1.2, n), rng.uniform(-0.9, 0.9, n), rng.uniform(0.8, 3.5, n)], 1)
    pc[n // 2:n // 2 + 400] = pc[:400]                                  # duplicates: equal zn whatever the rounding
    nc = np.tile([0.0, 0.0, -1.0], (n, 1))
    pose = rotated_pose()
    pw, nw = to_world(pose, pc, nc)
    store = np.zeros((n, 12), np.float32)
    store[:, 0:3] = pw; store[:, 3] = 20; store[:, 4] = 0x808080; store[:, 6] = 1; store[:, 7] = TICK; store[:, 8:11] = nw; store[:, 11] = 0.003
    depth, rgb = frame("zero")
    return Case("index_general", "index", store, pose, depth, rgb, {}, {"duplicates": 400})


# ======================================================================================================================================
# clean: k_clean_p1 / k_clean_p2, the ordered compactions k_clean_compact (in place) and k_clean_scatter (ping-pong)
# ======================================================================================================================================
def clean_keep(store, time=TICK, conf=CONF, time_delta=None):
    """copy_unstable.vert's verdict for a surfel whose window counts nothing (no neighbour passes the window's tests)"""
    lt = store[:, 7].copy()
    lt[lt == -2] = time
    c = store[:, 3]
    keep = ~((lt == -1) | ((f32(time) - lt > 20) & (c < conf)))
    if time_delta is not None:
        keep |= (lt > 0) & (f32(time) - lt > f32(time_delta))
    return keep


def place(n, visible, rng):
    """positions under the identity pose: `visible` entries on a grid of pixels 4 apart (nothing else in their index-map window: the
    window counts stay 0), the others behind the camera (finished in clean's pass 1 without a window)"""
    pos = np.zeros((n, 3), np.float32)
    pos[:, 0] = rng.uniform(-1, 1, n); pos[:, 1] = rng.uniform(-1, 1, n); pos[:, 2] = rng.uniform(-2.0, -0.5, n)
    vi = np.flatnonzero(visible)
    g = np.arange(vi.size)
    px, py = 2 + 4 * (g % 159), 2 + 4 * (g // 159)
    Z = (1.0 + 0.0001 * (g % 3000)).astype(np.float32)
    pos[vi, 0] = ((px + 0.5 - 320.0) * Z / 528.0).astype(np.float32)
    pos[vi, 1] = ((py + 0.5 - 240.0) * Z / 528.0).astype(np.float32)
    pos[vi, 2] = Z
    return pos


def removal(n, pattern, rng):
    r = np.zeros(n, bool)
    if pattern == "none":
        pass
    elif pattern == "all":
        r[:] = True
    elif pattern == "first":
        r[:1] = True
    elif pattern == "last":
        r[n - 1:] = True
    elif pattern == "511_512_513":
        r[[i for i in (511, 512, 513) if i < n]] = True
    elif pattern == "every_other":
        r[::2] = True
    elif pattern == "runs":                      # destination ranges of the following sub-blocks straddle a 512-entry edge
        for a, b in ((300, 420), (1000, 1030), (1530, 1600), (2047, 2049)):
            r[a:min(b, n)] = True
    elif pattern.startswith("d"):
        r = rng.random(n) < int(pattern[1:]) / 100.0
    else:
        raise ValueError(pattern)
    return r


def clean_case(name, n, pattern, frame_kind, capacity=1_200_000, seed=0, max_visible=4000):
    rng = np.random.default_rng(seed)
    rem = removal(n, pattern, rng)
    visible = (np.arange(n) % 7 == 3) & (np.cumsum(np.arange(n) % 7 == 3) <= max_visible)
    store = np.zeros((n, 12), np.float32)
    store[:, 0:3] = place(n, visible, rng)
    store[:, 3] = 20.0; store[:, 4] = 0x406080; store[:, 6] = 1.0
    store[:, 7] = np.where(rem, -1.0, np.where(np.arange(n) % 3 == 0, -2.0, float(TICK)))
    store[:, 8:11] = (0.0, 0.0, -1.0); store[:, 11] = 0.002
    depth, rgb = frame(frame_kind)
    kept = int(clean_keep(store).sum())
    new = NEW_ON_PLANE if frame_kind == "plane" else 0
    claims = {"count": n, "removed": int(rem.sum()), "pattern": pattern, "frame": frame_kind, "visible": int(visible.sum()),
              "clamped": int(kept + new > capacity), "full": int(n == capacity)}
    if pattern == "511_512_513":
        claims["removed_at_512_edge"] = int(rem[511:514].sum())
    return Case(name, "clean", store, IDENT, depth, rgb, {"capacityGlobal": capacity}, claims, min(kept + new, capacity), rem)


def clean_attrs():
    """the attribute tests of copy_unstable.vert: lastTime -1 / -2, age 20 / 21 against conf == threshold, one ulp below, above;
    visible surfels (window) and surfels behind the camera (pass 1)"""
    rows, claims = [], {}
    lo = nxt(CONF, 0)
    spec = [(-1.0, 20.0, "last_minus1"), (-2.0, 20.0, "last_minus2"), (-2.0, lo, "last_minus2_lowconf"),
            (TICK - 20, lo, "age20_conf_below"), (TICK - 20, CONF, "age20_conf_eq"),
            (TICK - 21, CONF, "age21_conf_eq"), (TICK - 21, lo, "age21_conf_below"), (TICK - 21, 10.5, "age21_conf_above")]
    vis = []
    for rep in range(3):
        for last, conf, key in spec:
            for v in (True, False):
                s = surfel(0, 0, 0, conf=conf, last=last); rows.append(s); vis.append(v)
                claims[key] = claims.get(key, 0) + 1
    store = np.stack(rows)
    visible = np.array(vis)
    store[:, 0:3] = place(len(rows), visible, np.random.default_rng(1))
    claims["visible"] = int(visible.sum()); claims["behind_camera"] = int((~visible).sum())
    depth, rgb = frame("zero")
    return Case("clean_attrs", "clean", store, IDENT, depth, rgb, {"capacityGlobal": 400000}, claims, int(clean_keep(store).sum()))


def clean_cases():
    cases = [clean_attrs()]
    for n, pat in ((0, "none"), (1, "first"), (511, "every_other"), (512, "last"), (513, "511_512_513")):
        for fk in ("zero", "plane"):
            cases.append(clean_case(f"clean_n{n}_{pat}_{fk}", n, pat, fk, seed=n))
    for pat in ("none", "all", "first", "last", "511_512_513", "every_other", "runs", "d1", "d50", "d99"):
        cases.append(clean_case(f"clean_n3000_{pat}", 3000, pat, "zero", seed=7))
    cases.append(clean_case("clean_n3000_runs_plane", 3000, "runs", "plane", seed=8))
    cases.append(clean_case("clean_clamp_plane", 3000, "d50", "plane", capacity=3000 + 5000, seed=9))
    cases.append(clean_case("clean_full_zero", 3000, "none", "zero", capacity=3000, seed=10))
    cases.append(clean_case("clean_full_plane", 3000, "d1", "plane", capacity=3000, seed=10))
    return cases


def clean_big():
    """the two ~1.1 M stores: 1 % removed with a plane frame, count + new > capacity (the clamp); and the first entry removed with a
    zero-depth frame (every sub-block moves down by one: the longest chain of hand-overs in the in-place compaction)"""
    return [clean_case("clean_big_d1_plane_clamp", BIG_N, "d1", "plane", capacity=1_150_000, seed=12),
            clean_case("clean_big_first_zero", BIG_N, "first", "zero", capacity=1_150_000, seed=13)]


# ======================================================================================================================================
# splat: k_splat_project / k_splat_resolve
# ======================================================================================================================================
def _radius_for_size(target, X, Y, Z, n=(0.0, 0.0, -1.0), r0=None):
    """float32 radius whose sprite has exactly `target` pixels (the oracle's size), or None: bisection over the float32 radii between
    r0 / 2 and 2 r0 (the size grows with the radius) for the smallest radius whose size reaches the target"""
    target = f32(target)
    if r0 is None:
        r0 = float(target) * float(Z) / (2 * np.sqrt(2) * 528.0)
    s = surfel(X, Y, Z, n=n, rad=0.0)

    def size(b):
        s[11] = np.int32(b).view(np.float32)
        return splat_extent(s).size

    lo, hi = int(f32(r0 / 2).view(np.int32)), int(f32(r0 * 2).view(np.int32))
    if size(lo) == target:                       # the lower clamp (size 1)
        return np.int32(lo).view(np.float32)
    if not size(lo) < target <= size(hi):
        return None
    while hi - lo > 1:
        m = (lo + hi) // 2
        if size(m) < target:
            lo = m
        else:
            hi = m
    return np.int32(hi).view(np.float32) if size(hi) == target else None


def splat_edges():
    rows, claims = [], {}

    def add(key, s):
        rows.append(s); claims[key] = claims.get(key, 0) + 1

    # two sprites over the whole image, behind everything else: raw size above 2047 (clamped) and just below it
    Zb = f32(19.0)
    r = _radius_for_size(2047, 0, 0, Zb)
    add("size_2047", surfel(0, 0, Zb, rad=r))
    add("size_above_2047", surfel(0, 0, f32(19.5), rad=f32(40.0)))
    add("size_below_2047", surfel(0, 0, f32(19.25), rad=nxt(_radius_for_size(2046, 0, 0, f32(19.25)), 0)))
    # R-PC: centres exactly on the viewport edges and one step outside
    Z = f32(2.0625)
    for tgt, key in [(0, "pc_x0"), (W, "pc_xW")]:
        X = solve(tgt, Z, FX, CX)
        add(key, surfel(X, f32(0.3), Z, rad=0.006))
        Xo = X
        while proj(Xo, Z, FX, CX) == f32(tgt):
            Xo = nxt(Xo, -np.inf if tgt == 0 else np.inf)
        add(key + "_outside", surfel(Xo, f32(0.3), Z, rad=0.006))
    for tgt, key in [(0, "pc_y0"), (H, "pc_yH")]:
        Y = solve(tgt, Z, FY, CY)
        add(key, surfel(f32(-0.4), Y, Z, rad=0.006))
        Yo = Y
        while proj(Yo, Z, FY, CY) == f32(tgt):
            Yo = nxt(Yo, -np.inf if tgt == 0 else np.inf)
        add(key + "_outside", surfel(f32(-0.4), Yo, Z, rad=0.006))
    # R-PR: camera-facing sprites of exact integer size centred on an integer (odd sizes) or half-integer (even sizes): every range
    # endpoint is a pixel centre; size 1 from a raw size below 1 and from a raw size of exactly 1
    for i, size in enumerate((1, 2, 3, 4, 5, 7, 9, 16)):
        Zs = f32(2.0)
        cxw = 60 + 30 * i + (0.5 if size % 2 == 0 else 0.0)
        X = solve(f32(cxw), Zs, FX, CX); Y = solve(f32(150 + (0.5 if size % 2 == 0 else 0.0)), Zs, FY, CY)
        rr = _radius_for_size(size, X, Y, Zs)
        if rr is None:
            raise AssertionError(f"no radius gives a sprite of exactly {size} pixels")
        add("rpr_exact_size", surfel(X, Y, Zs, rad=rr))
    add("size_raw_below_1", surfel(solve(f32(320), f32(2.0), FX, CX), solve(f32(200), f32(2.0), FY, CY), f32(2.0), rad=1e-5))
    # R-PR evaluated in fp32 (DESIGN section 4): the sums xw +- s/2 round where s/2 carries finer bits than the sum's ulp.  Centre on 300,
    # far behind the other sprites: size 199 - 2^-16 puts xw - s/2 at 200.5 + 2^-17, which rounds onto the centre 200.5 (pixel 200 in the
    # range although the exact rule leaves it out); size 199 + 2^-15 puts xw + s/2 at 399.5 + 2^-16, which rounds onto 399.5 (pixel 399
    # out although the exact rule takes it)
    for size, yc, key in ((f32(199 - 2.0 ** -16), 150, "rpr_fp32_tie_lo"), (f32(199 + 2.0 ** -15), 350, "rpr_fp32_tie_hi")):
        for k in range(400):
            Zt = f32(15.0 + k / 128.0)
            X = solve(f32(300), Zt, FX, CX)
            rr = None if X is None else _radius_for_size(size, X, f32((yc - 240.0) * float(Zt) / 528.0), Zt)
            if rr is not None:
                add(key, surfel(X, f32((yc - 240.0) * float(Zt) / 528.0), Zt, rad=rr))
                break
        else:
            raise AssertionError(f"no radius gives a sprite of exactly {size!r} pixels at xw == 300")
    # grazing incidence: |dot(l, n)| at 1e-1 .. 1e-7 for the ray of one pixel of the sprite
    for i, e in enumerate((1e-1, 1e-3, 1e-5, 1e-7)):
        px, py = 100 + 120 * i, 420
        l = np.array([(px + 0.5 - 320.0) / 528.0, (py + 0.5 - 240.0) / 528.0, 1.0]); l /= np.linalg.norm(l)
        u = np.cross(l, [0.0, 1.0, 0.0]); u /= np.linalg.norm(u)
        n = np.sqrt(1 - e * e) * u - e * l
        p = l * (2.0 / l[2])
        add(f"grazing_{e:.0e}", surfel(p[0], p[1], p[2], n=tuple(n), rad=0.02))
    # disc rim: dot(d, d) == rad^2 exactly at one pixel, and one ulp either side
    rim = {"rim_eq": 0, "rim_out": 0, "rim_in": 0}
    for k in range(40):
        if min(rim.values()) >= 3:
            break
        px, py = 30 + 14 * k, 30 + (k % 3) * 12
        nrm = (0.3, 0.2, -float(np.sqrt(1 - 0.13)))
        Zr = f32(1.7)
        X0 = f32((px + 0.5 + 0.8 - 320.0) * float(Zr) / 528.0); Y0 = f32((py + 0.5 + 0.3 - 240.0) * float(Zr) / 528.0)
        X = X0
        for _ in range(64):
            s = surfel(X, Y0, Zr, n=nrm, rad=0.01)
            sp = splat_extent(s)
            dd, _ = disc_dd(sp, px, py)
            r = f32(np.sqrt(dd, dtype=np.float32))
            for rc in (nxt(r, 0), r, nxt(r)):
                r2 = f32(rc * rc)
                key = "rim_eq" if r2 == dd else ("rim_out" if nxt(r2) == dd else ("rim_in" if nxt(r2, 0) == dd else None))
                if key and rim[key] < 3:
                    s2 = s.copy(); s2[11] = rc
                    sp2 = splat_extent(s2)
                    if sp2.ok and sp2.x0 <= px <= sp2.x1 and sp2.y0 <= py <= sp2.y1 and disc_dd(sp2, px, py)[0] == dd:
                        rim[key] += 1; rows.append(s2)
            X = nxt(X)
    claims.update(rim)
    # depth ties: coincident surfels (id order decides), and pairs one ulp apart with the nearer one later in the store
    for i in range(6):
        add("coincident", surfel(f32(0.3), f32(0.35), f32(2.2), rad=0.004))
    for i in range(4):
        Zp = f32(2.4 + 0.01 * i)
        X, Y = f32(-0.5 + 0.1 * i), f32(0.2)
        rows.append(surfel(X, Y, Zp, rad=0.005)); add("ulp_pair_nearer_later", surfel(X, Y, nxt(Zp, 0), rad=0.005))
    # fragment depth at the far plane: centre depth == maxDepth (fd == 1 at the centre), one ulp below, one ulp above (rejected)
    for Zf, key in [(MAXD, "z_maxdepth"), (nxt(MAXD, 0), "z_maxdepth_minus_ulp"), (nxt(MAXD), "z_maxdepth_plus_ulp")]:
        add(key, surfel(f32(-3.0), f32(-2.0), Zf, rad=0.05))
    # confidence at the threshold and one ulp below; last seen at maxTime and one frame later
    add("conf_eq_threshold", surfel(f32(0.5), f32(-0.6), f32(2.6), conf=CONF, rad=0.004))
    add("conf_below_threshold", surfel(f32(0.52), f32(-0.6), f32(2.6), conf=nxt(CONF, 0), rad=0.004))
    add("last_eq_maxtime", surfel(f32(0.6), f32(-0.6), f32(2.6), last=TICK, rad=0.004))
    add("last_after_maxtime", surfel(f32(0.62), f32(-0.6), f32(2.6), last=TICK + 1, rad=0.004))
    # 48 coincident 24-pixel sprites: every fragment passes the pre-tests, the per-warp queue of the exact path overflows many times
    rq = _radius_for_size(24, f32(0.9), f32(0.9), f32(2.5))
    for i in range(48):
        add("queue_stack", surfel(f32(0.9), f32(0.9), f32(2.5), rad=rq))
    store = np.stack(rows)
    depth, rgb = frame("zero")
    return Case("splat_edges", "splat", store, IDENT, depth, rgb, {}, claims)


def splat_rpr_overshoot(seed):
    """R-PR's open upper end where the disc reaches past the sprite: a tilted disc off the optical axis, close to the camera, whose near
    half projects beyond xw + s/2.  The centre projects exactly onto an integer and the radius is searched until the size is an exact
    odd integer, so xw + s/2 is exactly the centre of the column after the range; some pixels of that column pass the disc test and
    must stay undrawn.  One sprite per case: another sprite in front of it could hide that column."""
    rng = np.random.default_rng(seed)
    for _ in range(4000):
        th = rng.uniform(0.4, 0.9); phi = np.pi + rng.uniform(-0.7, 0.7)
        n = (float(np.sin(th) * np.cos(phi)), float(np.sin(th) * np.sin(phi)), float(-np.cos(th)))
        Z = f32(rng.uniform(0.5, 3.0))
        X = solve(f32(int(rng.integers(330, 480))), Z, FX, CX)
        if X is None:
            continue
        Y = f32(rng.uniform(-0.15, 0.15) * float(Z)); r0 = f32(rng.uniform(0.15, 0.35) * float(Z))
        sp = splat_extent(surfel(X, Y, Z, n=n, rad=r0))
        if not sp.ok:
            continue
        size = int(np.floor(sp.size)) | 1
        rr = _radius_for_size(size, X, Y, Z, n=n, r0=float(r0))
        if rr is None:
            continue
        s = surfel(X, Y, Z, n=n, rad=rr)
        sp = splat_extent(s)
        col = sp.x1 + 1
        if col >= W or float(sp.xw) + float(sp.size) / 2 != col + 0.5:
            continue
        if any(np.less_equal(*disc_dd(sp, col, py)) for py in range(sp.y0, sp.y1 + 1)):
            depth, rgb = frame("zero")
            return Case(f"splat_rpr_overshoot_{seed}", "splat", s[None, :].copy(), IDENT, depth, rgb, {}, {"rpr_hi_edge_in_disc": 1})
    raise AssertionError("no tilted disc reaches past its sprite at an exact pixel centre")


def splat_count(n):
    """n random surfels under a rotated pose: the bulk copy of the last round of positions is short (n % 128)"""
    rng = np.random.default_rng(100 + n)
    pc = np.stack([rng.uniform(-1.0, 1.0, n), rng.uniform(-0.8, 0.8, n), rng.uniform(0.8, 4.0, n)], 1)
    nc = np.stack([rng.uniform(-0.3, 0.3, n), rng.uniform(-0.3, 0.3, n), -np.ones(n)], 1)
    nc /= np.linalg.norm(nc, axis=1, keepdims=True)
    pose = rotated_pose(4)
    pw, nw = to_world(pose, pc, nc)
    store = np.zeros((n, 12), np.float32)
    store[:, 0:3] = pw; store[:, 3] = 20; store[:, 4] = rng.integers(0, 1 << 24, n); store[:, 6] = 1; store[:, 7] = TICK
    store[:, 8:11] = nw; store[:, 11] = rng.uniform(0.002, 0.03, n)
    depth, rgb = frame("zero")
    return Case(f"splat_n{n}", "splat", store, pose, depth, rgb, {}, {"count": n, "tail": n % 128})


# ======================================================================================================================================
# finite timeDelta: the time gates at equality in the index map (drawn), clean (no window: the fused noWindow path) and splat
# ======================================================================================================================================
TIME_DELTA = 5


def time_gates():
    rows, vis, claims = [], [], {}
    for last, key in [(TICK - TIME_DELTA, "dt_eq"), (TICK - TIME_DELTA - 1, "dt_above"), (TICK - TIME_DELTA + 1, "dt_below"),
                      (TICK - 25, "dt_old_lowconf"), (-2.0, "last_minus2")]:
        for rep in range(6):
            for v in (True, False):
                rows.append(surfel(0, 0, 0, conf=(5.0 if key == "dt_old_lowconf" else 20.0), last=last)); vis.append(v)
                claims[key] = claims.get(key, 0) + 1
    store = np.stack(rows)
    visible = np.array(vis)
    store[:, 0:3] = place(len(rows), visible, np.random.default_rng(2))
    claims["visible"] = int(visible.sum())
    depth, rgb = frame("zero")
    return Case("time_gates", "time", store, IDENT, depth, rgb, {"timeDelta": TIME_DELTA, "capacityGlobal": 400000}, claims,
                int(clean_keep(store, time_delta=TIME_DELTA).sum()))


@functools.lru_cache(maxsize=None)
def small_cases():
    return [index_edges(), index_general(), *clean_cases(), splat_edges(), splat_rpr_overshoot(1), splat_rpr_overshoot(2), *[splat_count(n) for n in (1, 127, 128, 129, 1000)], time_gates()]


@functools.lru_cache(maxsize=None)
def big_cases():
    return clean_big()


def all_cases():
    return [*small_cases(), *big_cases()]
