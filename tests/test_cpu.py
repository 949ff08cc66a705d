"""CPU-side tests (no GPU): the oracle against analytic expectations and the committed
golden vectors, the written raster / ordering rules, the host logic, and that the C-ABI
library loads and exports every symbol include/maskfusion_b200.h declares."""
from __future__ import annotations

import ctypes as C
import os
import re

import numpy as np
import pytest

from tests import oracle_lib as ol

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


# ------------------------------------------------------------------------------- helpers
def surfel(pos, conf=20.0, color=0x808080, init_t=1, last_t=1, n=(0, 0, -1), r=0.01):
    return np.array([pos[0], pos[1], pos[2], conf, float(color), 0, init_t, last_t, n[0], n[1], n[2], r], np.float32)


CAM = (528.0, 528.0, 320.0, 240.0)
W, H = 640, 480
I4 = np.eye(4, dtype=np.float32)


def predict_indices(surfels, pose=I4, max_depth=20.0, time=2, time_delta=1 << 30):
    L = ol.lib()
    s = np.ascontiguousarray(surfels, np.float32)
    idx = np.zeros((H, W), np.uint32); vc = np.zeros((H, W, 4), np.float32); ct = np.zeros((H, W, 4), np.float32); nr = np.zeros((H, W, 4), np.float32)
    L.orc_predict_indices(ol.ptr(s), s.shape[0], ol.ptr(np.ascontiguousarray(pose)), ol.cam(*CAM), W, H, C.c_float(max_depth), time, time_delta,
                          ol.ptr(idx), ol.ptr(vc), ol.ptr(ct), ol.ptr(nr))
    return idx, vc, ct, nr


# ------------------------------------------------------------------------------- maths
def test_deterministic_exp_acos_accuracy():
    L = ol.lib()
    xs = np.linspace(-80, 5, 4001).astype(np.float32)
    ys = np.array([L.orc_expf(float(x)) for x in xs])
    assert np.max(np.abs(ys - np.exp(xs.astype(np.float64))) / np.exp(xs.astype(np.float64))) < 2e-7
    assert L.orc_expf(-200.0) == 0.0
    xa = np.linspace(-1, 1, 2001).astype(np.float32)
    ya = np.array([L.orc_acosf(float(x)) for x in xa])
    assert np.max(np.abs(ya - np.arccos(xa.astype(np.float64)))) < 1e-6
    assert np.isnan(L.orc_acosf(1.5))


def test_ldlt_and_rodrigues():
    L = ol.lib()
    rng = np.random.default_rng(0)
    M = rng.normal(size=(6, 6)); A = M @ M.T + 6 * np.eye(6); b = rng.normal(size=6); x = np.zeros(6)
    L.orc_ldlt_solve(ol.ptr(A), ol.ptr(b), 6, ol.ptr(x))
    assert np.allclose(x, np.linalg.solve(A, b), rtol=1e-10, atol=1e-12)
    Z = np.zeros((6, 6)); L.orc_ldlt_solve(ol.ptr(Z), ol.ptr(b), 6, ol.ptr(x))
    assert np.all(x == 0)                       # Eigen: singular pivots solve to 0 (no correspondences => no motion)
    w = np.array([0.1, -0.2, 0.05]); R = np.zeros(9)
    L.orc_rodrigues(ol.ptr(w), ol.ptr(R)); R = R.reshape(3, 3)
    assert np.allclose(R @ R.T, np.eye(3), atol=1e-12) and np.isclose(np.trace(R), 1 + 2 * np.cos(np.linalg.norm(w)))


# ------------------------------------------------------------------------------- maps
def test_vmap_nmap_conventions():
    """integer pixel coordinates (no +0.5), invalid => NaN in x, last row/col of nmap NaN (cudafuncs.cu:109-189)"""
    L = ol.lib()
    d = np.full((H, W), 2.0, np.float32); d[10, 10] = 0; d[20, 20] = 9.0
    v = np.zeros((3, H, W), np.float32); n = np.zeros((3, H, W), np.float32)
    L.orc_vmap(ol.ptr(d), W, H, ol.cam(*CAM), C.c_float(4.0), ol.ptr(v)); L.orc_nmap(ol.ptr(v), W, H, ol.ptr(n))
    assert v[0, 240, 320] == 0 and v[1, 240, 320] == 0 and v[2, 240, 320] == 2.0
    assert np.isclose(v[0, 240, 321], 2.0 / 528.0)
    assert np.isnan(v[0, 10, 10]) and v[2, 10, 10] == 0 and np.isnan(v[0, 20, 20])
    assert np.isnan(n[0, :, W - 1]).all() and np.isnan(n[0, H - 1, :]).all()
    assert np.isnan(n[0, 10, 9]) and np.isnan(n[0, 9, 10])           # neighbours of an invalid vertex
    assert np.allclose([n[0, 100, 100], n[1, 100, 100], n[2, 100, 100]], [0, 0, 1], atol=1e-6)


def test_pyramid_quirks():
    """N9: window clamp excludes the last column/row; int weight sum; uchar zeros skipped"""
    L = ol.lib()
    src = np.arange(8 * 8, dtype=np.float32).reshape(8, 8); dst = np.zeros((4, 4), np.float32)
    L.orc_pyrdown_gauss_f(ol.ptr(src), 8, 8, ol.ptr(dst))
    # centre pixel (1,1): full 5x5 window [0..4]x[0..4]
    g = np.array([1, 4, 6, 4, 1], np.float32); k = np.outer(g, g)
    ty, tx = 5, 5
    acc = 0.0
    for cy in range(0, 5):
        for cx in range(0, 5):
            acc += src[cy, cx] * k[ty - cy - 1, tx - cx - 1]
    assert np.isclose(dst[1, 1], acc / 256.0)
    # last output column: tx clamps to cols-1 = 7 -> window [4,7): column 7 never read
    src2 = np.ones((8, 8), np.float32); src2[:, 7] = 1000.0
    L.orc_pyrdown_gauss_f(ol.ptr(src2), 8, 8, ol.ptr(dst))
    assert np.all(dst[:3, 3] == 1.0)
    u = np.zeros((8, 8), np.uint8); u[2, 2] = 200; du = np.zeros((4, 4), np.uint8)
    L.orc_pyrdown_gauss_u8(ol.ptr(u), 8, 8, ol.ptr(du))
    assert du[1, 1] == 200 and du[3, 3] == 0


# ------------------------------------------------------------------------------- raster rules
def test_index_map_depth_test_and_tie_rule():
    """N2: pixel = floor(projection); nearest z wins; equal z -> lowest surfel id; id 0 reads as empty"""
    s = np.stack([surfel((0.0, 0.0, 2.0)),            # id 0 -> pixel (320,240)
                  surfel((0.5, 0.0, 2.0)),            # id 1 -> pixel (452,240)
                  surfel((0.5, 0.0, 1.5 * 2.0 / 1.5)),  # id 2 same pixel, same z -> loses the tie to id 1
                  surfel((0.25, 0.0, 1.0)),           # id 3 -> pixel (452,240), nearer -> wins
                  surfel((0.0, 0.0, 25.0)),           # beyond maxDepth
                  surfel((0.0, 0.0, -1.0))])          # behind the camera
    idx, vc, ct, nr = predict_indices(s)
    assert idx[240, 320] == 0 and vc[240, 320, 2] == 2.0      # surfel 0 occupies the pixel but reads as "empty"
    assert idx[240, 452] == 3 and vc[240, 452, 2] == 1.0
    idx2, *_ = predict_indices(s[:3])
    assert idx2[240, 452] == 1
    assert (idx > 0).sum() == 1


def test_index_map_time_window():
    s = np.stack([surfel((0, 0, 2.0)), surfel((0.5, 0, 2.0), last_t=1)])
    idx, *_ = predict_indices(s, time=100, time_delta=10)
    assert (idx > 0).sum() == 0
    idx, *_ = predict_indices(s, time=100, time_delta=200)
    assert idx[240, 452] == 1


def test_fuse_update_rule_and_collision_order():
    """update.vert:57-95; N4: the first pixel in x-major order owns the surfel"""
    L = ol.lib()
    s = np.stack([surfel((0, 0, 2.0), conf=1.0, r=0.01), surfel((1, 0, 2.0), conf=2.0, r=0.01)]).copy()
    upd = np.zeros((W, H), np.uint8); best = np.zeros((W, H), np.uint32); meas = np.zeros((W, H, 12), np.float32)
    # two pixels claim surfel 1: x-major order => (x=5,y=7) precedes (x=6,y=0)
    upd[5, 7] = 1; best[5, 7] = 1; meas[5, 7] = surfel((1.2, 0, 2.0), conf=2.0, r=0.012, color=0x404040); meas[5, 7, 7] = -1
    upd[6, 0] = 1; best[6, 0] = 1; meas[6, 0] = surfel((9, 9, 9), conf=2.0, r=0.012); meas[6, 0, 7] = -1
    # radius too large => only confidence / time change
    upd[9, 9] = 1; best[9, 9] = 0; meas[9, 9] = surfel((5, 5, 5), conf=0.5, r=0.02); meas[9, 9, 7] = -1
    L.orc_fuse_update(ol.ptr(s), 2, ol.ptr(upd), ol.ptr(best), ol.ptr(meas), W, H, 7)
    assert np.allclose(s[1, :3], [1.1, 0, 2.0]) and s[1, 3] == 4.0 and s[1, 7] == 7 and np.isclose(s[1, 11], 0.011)
    assert np.allclose(s[0, :3], [0, 0, 2.0]) and s[0, 3] == 1.5 and s[0, 7] == 7 and s[0, 11] == np.float32(0.01)
    assert int(s[1, 4]) == 0x606060


def test_clean_ordering_and_unstable_removal():
    """N5: survivors keep buffer order, new vertices follow in x-major pixel order; N6: drop if time-t>20 && conf<thr"""
    L = ol.lib()
    s = np.stack([surfel((0, 0, 2.0), conf=20, last_t=30), surfel((0.1, 0, 2.0), conf=1.0, last_t=2),   # unstable for > 20 frames -> dropped
                  surfel((0.2, 0, 2.0), conf=1.0, last_t=25), surfel((0.3, 0, 2.0), conf=30, last_t=1)])
    upd = np.zeros((W, H), np.uint8); meas = np.zeros((W, H, 12), np.float32)
    upd[300, 10] = 2; meas[300, 10] = surfel((0.5, 0.5, 2.0), conf=0.7); meas[300, 10, 7] = -2
    upd[20, 400] = 2; meas[20, 400] = surfel((-0.5, 0.5, 2.0), conf=0.8); meas[20, 400, 7] = -2
    upd[100, 100] = 1; meas[100, 100] = surfel((0, 0.5, 2.0)); meas[100, 100, 7] = -1                   # merge record: never copied
    idx = np.zeros((H, W), np.uint32); z4 = np.zeros((H, W, 4), np.float32)
    depth = np.zeros((H, W), np.float32); mask = np.zeros((H, W), np.uint8)
    out = np.zeros((16, 12), np.float32)
    n = L.orc_clean(ol.ptr(s), 4, ol.ptr(upd), ol.ptr(meas), ol.ptr(idx), ol.ptr(z4), ol.ptr(z4), ol.ptr(depth), ol.ptr(mask), ol.ptr(I4),
                    ol.cam(*CAM), W, H, 30, 1 << 30, C.c_float(10.0), C.c_float(0.1), 0, ol.ptr(out), 16)
    assert n == 5
    assert np.allclose(out[:3, 0], [0, 0.2, 0.3])
    assert np.allclose(out[3, :2], [-0.5, 0.5]) and np.allclose(out[4, :2], [0.5, 0.5])    # x=20 precedes x=300
    assert out[3, 7] == 30 and out[4, 7] == 30                                            # -2 -> time


def test_splat_point_and_disc_rule():
    """combo_splat.frag: ray/disc intersection inside radius; vertex at the pixel centre (+0.5, N1)"""
    L = ol.lib()
    s = np.stack([surfel((0.001, 0.001, 2.0), conf=20, r=0.02)])
    im = np.zeros((H, W, 4), np.uint8); vc = np.zeros((H, W, 4), np.float32); nr = np.zeros((H, W, 4), np.float32); tt = np.zeros((H, W), np.uint16)
    L.orc_combined_predict(ol.ptr(s), 1, ol.ptr(I4), ol.cam(*CAM), W, H, C.c_float(20.0), C.c_float(10.0), 2, 2, 1 << 30,
                           ol.ptr(im), ol.ptr(vc), ol.ptr(nr), ol.ptr(tt))
    hit = vc[..., 2] > 0
    assert hit.sum() > 20                               # r=2cm at 2 m ~ 5 px radius
    ys, xs = np.nonzero(hit)
    assert abs(xs.mean() - 320.0) < 1.5 and abs(ys.mean() - 240.0) < 1.5
    y, x = ys[0], xs[0]
    assert np.isclose(vc[y, x, 0], (x + 0.5 - 320.0) * vc[y, x, 2] / 528.0, rtol=1e-5)
    assert np.all(np.hypot(vc[hit][:, 0] - 0.001, vc[hit][:, 1] - 0.001) <= 0.02 + 1e-6)
    assert im[y, x, 3] == 255 and tuple(im[y, x, :3]) == (128, 128, 128)
    # below the confidence threshold nothing is drawn (splat.vert:58)
    s[0, 3] = 5.0
    L.orc_combined_predict(ol.ptr(s), 1, ol.ptr(I4), ol.cam(*CAM), W, H, C.c_float(20.0), C.c_float(10.0), 2, 2, 1 << 30,
                           ol.ptr(im), ol.ptr(vc), ol.ptr(nr), ol.ptr(tt))
    assert (vc[..., 2] > 0).sum() == 0


# ------------------------------------------------------------------------------- odometry
def test_icp_recovers_small_motion_without_filtering():
    """point-to-plane GN on exact synthetic depth converges to the ground-truth increment (< 0.05 mm)"""
    from maskfusion_b200.synth import SynthScene
    L = ol.lib()
    sc = SynthScene(W, H, n_objects=0, seed=0)
    cam = ol.cam(*CAM)

    def maps(d):
        v = np.zeros((3, H, W), np.float32); n = np.zeros((3, H, W), np.float32)
        L.orc_vmap(ol.ptr(d), W, H, cam, C.c_float(4.0), ol.ptr(v)); L.orc_nmap(ol.ptr(v), W, H, ol.ptr(n))
        return v, n
    sc.render(0); d0 = sc.last_depth_exact.copy(); T0 = sc.camera_pose(0)
    sc.render(1); d1 = sc.last_depth_exact.copy(); T1 = sc.camera_pose(1)
    gt = np.linalg.inv(T0) @ T1
    vg, ng = maps(d0); v1, n1 = maps(d1)
    I3 = np.eye(3, dtype=np.float32).ravel().copy(); z3 = np.zeros(3, np.float32)
    res = np.eye(4)
    for _ in range(8):
        cur = np.linalg.inv(res)
        Rc = np.ascontiguousarray(cur[:3, :3], np.float32).ravel(); tc = np.ascontiguousarray(cur[:3, 3], np.float32)
        out = np.zeros(29)
        L.orc_icp_step(ol.ptr(Rc), ol.ptr(tc), ol.ptr(v1), ol.ptr(n1), ol.ptr(I3), ol.ptr(z3), cam, ol.ptr(vg), ol.ptr(ng),
                       C.c_float(0.1), C.c_float(np.sin(np.radians(20))), W, H, ol.ptr(out))
        A = np.zeros((6, 6)); b = np.zeros(6); k = 0
        for i in range(6):
            for j in range(i, 7):
                if j == 6: b[i] = out[k]
                else: A[i, j] = A[j, i] = out[k]
                k += 1
        x = np.zeros(6); L.orc_ldlt_solve(ol.ptr(A), ol.ptr(b), 6, ol.ptr(x))
        up = np.eye(4); Rr = np.zeros(9); L.orc_rodrigues(ol.ptr(x[3:].copy()), ol.ptr(Rr)); up[:3, :3] = Rr.reshape(3, 3); up[:3, 3] = x[:3]
        res = up @ res
    est = np.linalg.inv(res)
    assert np.linalg.norm(est[:3, 3] - gt[:3, 3]) < 5e-5
    assert out[28] > 0.9 * W * H


def test_static_pipeline_matches_golden():
    """oracle regression pin: the committed golden vector was produced by tests/golden/make_golden.py"""
    from maskfusion_b200.synth import SynthScene
    g = np.load(os.path.join(ROOT, "tests", "golden", "static_icp_160x120.npz"))
    w, h = 160, 120
    sc = SynthScene(w, h, n_objects=0, seed=3)
    p = ol.OraclePipeline(ol.default_config(w, h, capacityGlobal=60000, icpWeight=100.0, so3=0))
    for t in range(int(g["nframes"])):
        rgb, depth, *_ = sc.render(t)
        p.process_frame(rgb, depth, t)
    assert p.count(0) == int(g["count"])
    assert np.array_equal(p.pose(0), g["pose"])
    assert np.array_equal(p.tex(0, "idx"), g["idx"])
    assert np.array_equal(p.surfels(0)[::97], g["surfels_97"])


def test_static_pipeline_tracks_camera():
    from maskfusion_b200.synth import SynthScene
    sc = SynthScene(W, H, n_objects=0, seed=0)
    T0 = sc.camera_pose(0)
    errs = {}
    for name, kw in (("icp", dict(icpWeight=100.0, so3=0)), ("gui", dict())):     # gui = GUI defaults: ICP+RGB (w=20), SO3
        p = ol.OraclePipeline(ol.default_config(W, H, capacityGlobal=500000, **kw))
        for t in range(4):
            rgb, depth, _, Tc, _ = sc.render(t)
            p.process_frame(rgb, depth, t)
        gt = np.linalg.inv(T0) @ Tc
        errs[name] = np.linalg.norm(p.pose(0)[:3, 3] - gt[:3, 3]) / np.linalg.norm(gt[:3, 3])
        assert p.count(0) > 300000
    # ICP only: ~8 % lag (bilateral-filter edge bias).  GUI defaults: A = A_rgb + w^2 A_icp, b = b_rgb + w b_icp with
    # MaskFusion's sigma = rgbSize makes every GN step ~1/w of the ICP step => ~35 % lag per frame in
    # frame-to-frame mode (documented in DESIGN.md "reference quirks"); the oracle reproduces it.
    assert errs["icp"] < 0.12, errs
    assert 0.2 < errs["gui"] < 0.5, errs


# ------------------------------------------------------------------------------- product library (no compute without a GPU)
def test_c_abi_exports_every_declared_symbol(product_lib):
    hdr = open(os.path.join(ROOT, "include", "maskfusion_b200.h")).read()
    names = set(re.findall(r"\b(mf_[a-z0-9_]+)\s*\(", hdr))
    names -= {"mf_config", "mf_context", "mf_klg"}
    L = product_lib.load_library()
    missing = [n for n in sorted(names) if not hasattr(L, n)]
    assert not missing, missing
    assert set(product_lib.EXPORTS) == names and len(product_lib.EXPORTS) == len(names)
    assert L.mf_abi_version() == 1


def test_config_defaults_match_oracle(product_lib):
    a = product_lib.default_config(640, 480); b = ol.default_config(640, 480)
    for f, _ in product_lib.Config._fields_:
        assert getattr(a, f) == getattr(b, f), f
    assert bytes(a) == bytes(b)


def test_no_cpu_fallback(product_lib):
    import torch
    if torch.cuda.is_available():
        pytest.skip("GPU present")
    with pytest.raises(product_lib.MFError, match="no CPU fallback"):
        product_lib.MaskFusion(product_lib.default_config(640, 480))


def test_klg_roundtrip_and_reader_quirks(product_lib, tmp_path):
    """layout KlgLogReader.cpp:29,53-89; N11: hasMore() hides the last frame; depth u16 mm * 0.001 via double"""
    n, w, h = 4, 64, 48
    rng = np.random.default_rng(0)
    d = rng.integers(0, 6000, (n, h, w)).astype(np.uint16); c = rng.integers(0, 255, (n, h, w, 3)).astype(np.uint8)
    ts = np.arange(n, dtype=np.int64) * 33333
    path = str(tmp_path / "t.klg")
    product_lib.write_klg(path, ts, d, c)
    raw = open(path, "rb").read()
    assert np.frombuffer(raw[:4], np.int32)[0] == n and len(raw) == 4 + n * (8 + 4 + 4 + w * h * 5)
    r = product_lib.KlgLogReader(path, w, h)
    assert r.getNumFrames() == n
    got = 0
    while r.hasMore():
        rgb, depth, t = r.getNext()
        assert t == ts[got] and np.array_equal(rgb, c[got])
        assert np.array_equal(depth, (d[got].astype(np.float64) * 0.001).astype(np.float32))
        got += 1
    assert got == n - 1
    r.close()
    r = product_lib.KlgLogReader(path, w, h, flipColors=True)
    rgb, _, _ = r.getNext()
    assert np.array_equal(rgb, c[0][..., ::-1])
    r.close()
    with pytest.raises(product_lib.MFError):
        product_lib.KlgLogReader(str(tmp_path / "missing.klg"), w, h)


def test_entry_scripts_compile():
    """bench.py / __graft_entry__.py / scripts are only executed on the GPU box: a syntax error there would cost a round"""
    import glob
    import py_compile
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    for f in [os.path.join(root, "bench.py"), os.path.join(root, "__graft_entry__.py")] + glob.glob(os.path.join(root, "scripts", "*.py")) + \
            glob.glob(os.path.join(root, "maskfusion_b200", "*.py")) + glob.glob(os.path.join(root, "tests", "*.py")):
        py_compile.compile(f, doraise=True)


def test_oracle_is_thread_count_invariant():
    """the oracle's OpenMP sections keep the sequential semantics (order-free 64-bit min for the depth tests, one thread per
    accumulator for the sums, ordered copy-out for the compaction): 1 thread and 5 threads must give the same bits"""
    import subprocess
    import sys
    code = (
        "import sys, hashlib, numpy as np\n"
        f"sys.path.insert(0, {ROOT!r})\n"
        "from tests import oracle_lib as ol\n"
        "from maskfusion_b200.synth import SynthScene\n"
        "sc = SynthScene(160, 120, n_objects=0, seed=5)\n"
        "p = ol.OraclePipeline(ol.default_config(160, 120, capacityGlobal=60000))\n"
        "for t in range(4):\n"
        "    rgb, depth, *_ = sc.render(t); p.process_frame(rgb, depth, t * 33333)\n"
        "print(hashlib.sha1(p.surfels(0).tobytes()).hexdigest(), hashlib.sha1(p.pose(0).tobytes()).hexdigest(), hashlib.sha1(p.tex(0, 'splatVertex').tobytes()).hexdigest(), p.count(0))\n")
    outs = []
    for n in ("1", "5"):
        env = dict(os.environ, OMP_NUM_THREADS=n)
        r = subprocess.run([sys.executable, "-c", code], capture_output=True, text=True, env=env, timeout=300)
        assert r.returncode == 0, r.stderr[-800:]
        outs.append(r.stdout.strip().splitlines()[-1])
    assert outs[0] == outs[1], outs


def test_oracle_opencv_restatements_match_cv2(oracle):
    """VERDICT r1 weak 3: the OpenCV semantics restated in oracle/orc_mfseg.c -- connectedComponentsWithStats(4-connectivity) and
    morphologyEx(MORPH_CLOSE, MORPH_ELLIPSE, iterations) -- against the cv2 that is importable here (4.13; upstream pins 3.4.1).
    Labels are compared up to a permutation (the reference's results do not depend on the numbering), stats exactly."""
    cv2 = pytest.importorskip("cv2")
    import ctypes as C
    L = oracle.lib()
    L.orc_connected_components4.restype = C.c_int
    L.orc_connected_components4.argtypes = [C.c_void_p, C.c_int, C.c_int, C.c_void_p, C.POINTER(C.POINTER(C.c_int32))]
    L.orc_morph_close_ellipse.argtypes = [C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_int]
    libc = C.CDLL(None)
    libc.free.argtypes = [C.c_void_p]
    rng = np.random.default_rng(3)
    for (W, H, p) in [(64, 48, 0.55), (97, 61, 0.7), (640, 480, 0.62), (33, 17, 0.9), (16, 16, 0.0), (16, 16, 1.0)]:
        img = (rng.random((H, W)) < p).astype(np.uint8) * 255
        if W == 640:                      # realistic: blobs with thin bridges
            yy, xx = np.mgrid[0:H, 0:W]
            img = (((np.sin(xx / 9.0) * np.cos(yy / 7.0) > -0.2) & (rng.random((H, W)) < 0.97)) * 255).astype(np.uint8)
        labels = np.zeros((H, W), np.int32)
        stats_p = C.POINTER(C.c_int32)()
        n = L.orc_connected_components4(oracle.ptr(img), W, H, oracle.ptr(labels), C.byref(stats_p))
        stats = np.ctypeslib.as_array(stats_p, shape=(n, 5)).copy()
        libc.free(stats_p)
        n_cv, lab_cv, stats_cv, _ = cv2.connectedComponentsWithStats(img, connectivity=4, ltype=cv2.CV_32S)
        assert n == n_cv, (W, H, n, n_cv)
        assert np.array_equal(labels == 0, lab_cv == 0)
        # one-to-one label correspondence
        pairs = np.unique(np.stack([labels.ravel(), lab_cv.ravel()], 1), axis=0)
        present = n if (labels == 0).any() else n - 1          # label 0 has no pixel when the image has no zero
        assert pairs.shape[0] == present and len(set(pairs[:, 0])) == present and len(set(pairs[:, 1])) == present
        remap = np.zeros(n, np.int64); remap[pairs[:, 0]] = pairs[:, 1]
        # stats columns: left, top, width, height, area (background row: cv2 reports the bounding box of the zero pixels too)
        assert np.array_equal(stats[1:], stats_cv[remap[1:]]), (W, H)
        assert stats[0, 4] == stats_cv[0, 4]
    for (W, H) in [(64, 48), (640, 480)]:
        seg = np.zeros((H, W), np.uint8)
        for k in range(1, 6):             # mask-id image: a few labelled blobs with holes and gaps, plus 255 (ignored) pixels
            cx, cy, r = rng.integers(8, W - 8), rng.integers(8, H - 8), rng.integers(4, max(5, H // 5))
            yy, xx = np.mgrid[0:H, 0:W]
            seg[(xx - cx) ** 2 + (yy - cy) ** 2 < r * r] = k
        seg[rng.random((H, W)) < 0.08] = 0
        seg[rng.random((H, W)) < 0.01] = 255
        for r in (0, 1, 2, 3, 5):
            for it in (0, 1, 2, 3):
                a = seg.copy()
                L.orc_morph_close_ellipse(oracle.ptr(a), W, H, r, it)
                el = cv2.getStructuringElement(cv2.MORPH_ELLIPSE, (2 * r + 1, 2 * r + 1), (r, r))
                ref = cv2.morphologyEx(seg, cv2.MORPH_CLOSE, el, anchor=(-1, -1), iterations=it) if it > 0 else seg
                assert np.array_equal(a, ref), (W, H, r, it, int((a != ref).sum()))


def test_mfseg_tail_thread_invariant_and_sane(oracle):
    """BASELINE configs[0] workload (one 640x480 frame through the CPU part of MfSegmentation::performSegmentation): the OpenMP
    split used for the all-cores timing gives the single-threaded result bit for bit, with and without the mask close"""
    fr = oracle.segmentation_frame()
    for it in (0, 2):
        s1, n1, h1, _ = oracle.run_mfseg_cpu(fr, threads=1, morphMaskIterations=it)
        s4, n4, h4, _ = oracle.run_mfseg_cpu(fr, threads=4, morphMaskIterations=it)
        assert n1 == n4 and h1 == h4 and np.array_equal(s1, s4)
        assert n1 > 5 and set(np.unique(s1)) >= {0, 1, 2, 3}           # background + the three instances mapped to their models


def test_warp_ldlt_scheme_is_bit_identical_to_the_sequential_routine(oracle):
    """The CUDA solver (csrc/mf_track.cu: ldltSolvePivWarp) distributes the oracle's pivoted LDL^T over the lanes of a warp: lane i owns
    row i of the FULL matrix, the trailing update writes both halves (the upper entry with the operand order of its mirror image) and the
    back substitution derives L[j][i] from the lane's own upper entries.  This emulates that data flow operation for operation in
    numpy float64 and checks the solution against orc_ldlt_solve BIT FOR BIT on SPD, ill-conditioned and singular systems -- the
    argument for why tracked trajectories can be identical, runnable without a GPU (the kernel itself is covered by the GPU tests)."""
    import ctypes as C
    L = oracle.lib()
    L.orc_ldlt_solve.argtypes = [C.c_void_p, C.c_void_p, C.c_int, C.c_void_p]
    tiny = np.finfo(np.float64).tiny

    def warp(Ain, b):
        n = len(b)
        a = [[np.float64(Ain[i][j]) for j in range(n)] for i in range(n)]
        perm = list(range(n)); kend = n
        for k in range(n):
            piv = k; best = abs(a[k][k])
            for i in range(k + 1, n):
                if abs(a[i][i]) > best:
                    best = abs(a[i][i]); piv = i
            if piv != k:
                a[k], a[piv] = a[piv], a[k]
                perm[k], perm[piv] = perm[piv], perm[k]
                for r in range(n):
                    a[r][k], a[r][piv] = a[r][piv], a[r][k]
            d = a[k][k]
            if abs(d) <= tiny:
                kend = k
                break
            for i in range(k + 1, n):
                a[i][k] = a[i][k] / d
            col = [a[j][k] for j in range(n)]
            for r in range(k + 1, n):
                ad = a[r][k] * d
                for j in range(k + 1, n):
                    a[r][j] = a[r][j] - ad * col[j] if j <= r else a[r][j] - (col[j] * d) * a[r][k]
        for i in range(kend, n):
            for j in range(kend, i):
                a[i][j] = np.float64(0)
        y = [np.float64(b[perm[i]]) for i in range(n)]
        for j in range(n - 1):
            for i in range(j + 1, n):
                if j < kend:
                    y[i] = y[i] - a[i][j] * y[j]
        for i in range(n):
            dd = a[i][i] if i < kend else np.float64(0)
            y[i] = y[i] / dd if abs(dd) > tiny else np.float64(0)
        for i in range(n - 2, -1, -1):
            if i < kend:
                for j in range(i + 1, n):
                    y[i] = y[i] - (a[i][j] / a[i][i]) * y[j]
        x = np.zeros(n)
        for i in range(n):
            x[perm[i]] = y[i]
        return x

    rng = np.random.default_rng(0)
    with np.errstate(all="ignore"):
        for trial in range(600):
            n = 6 if trial % 4 else 3
            m = int(rng.integers(n, 40))
            J = rng.normal(size=(m, n)) * rng.uniform(0.01, 10, size=(1, n))
            if trial % 7 == 0:
                J[:, rng.integers(0, n)] = 0
            if trial % 11 == 0:
                J[:, 1] = J[:, 0] * 2
            A = np.float64(np.float32(J.T @ J))
            for i in range(n):
                for j in range(i):
                    A[i][j] = A[j][i]
            b = np.float64(np.float32(J.T @ rng.normal(size=m)))
            A = np.ascontiguousarray(A); b = np.ascontiguousarray(b)
            xo = np.zeros(n)
            L.orc_ldlt_solve(A.ctypes.data, b.ctypes.data, n, xo.ctypes.data)
            assert np.array_equal(xo.view(np.uint64), warp(A, b).view(np.uint64)), trial


def test_track_shares_host_logic():
    """grid shares of the persistent tracking launch (mf_track_shares): every CTA is dealt at most once, light models >= 4 CTAs, a heavy
    model gets ~ratio times a light one, equal shares without both kinds in the batch"""
    import ctypes as C
    import maskfusion_b200 as mfb
    L = mfb.load_library()

    def shares(n, mask, total=148, ratio=2):
        out = (C.c_int * 32)()
        assert L.mf_track_shares(n, mask, total, ratio, out) == 0
        return list(out[:n])
    assert shares(1, 0) == [148]
    assert shares(3, 0) == [49, 49, 49] and shares(3, 0b111) == [49, 49, 49]           # one kind only: equal
    s9 = shares(9, 0b111111110)                                                     # background + 8 objects
    assert s9[0] == 148 - 8 * s9[1] and all(x == s9[1] for x in s9[1:]) and s9[1] == 148 // 10 and sum(s9) <= 148
    s4 = shares(4, 0b1110)
    assert s4 == [148 - 3 * 29, 29, 29, 29]
    s17 = shares(17, 0x1fffe)                                                       # configs[4]: 16 objects + background
    assert min(s17) >= 4 and sum(s17) <= 148 and s17[0] > s17[1]
    for n in range(1, 33):
        for mask in (0, 1, (1 << n) - 2, 0x55555555 & ((1 << n) - 1)):
            for total in (132, 148, 160):
                s = shares(n, mask, total)
                assert min(s) >= 1 and sum(s) <= total, (n, mask, total, s)
    assert L.mf_track_shares(0, 0, 148, 2, (C.c_int * 32)()) != 0 and L.mf_track_shares(33, 0, 148, 2, (C.c_int * 32)()) != 0


def test_inplace_compaction_scheme_model():
    """Model of k_clean_compact's hand-over (DESIGN 3e) under random schedules: sub-blocks of B entries are taken in ticket order by a few
    resident workers; a sub-block loads its survivors, publishes `loaded`, and may store once the lower sub-blocks whose SOURCE range its
    destination range overlaps have published.  Checked: no store ever lands on a source entry that has not been loaded yet, nobody waits on
    a higher ticket (no deadlock), and the array ends as the ordered compaction."""
    rng = np.random.default_rng(3)
    B = 8
    for trial in range(300):
        n = int(rng.integers(1, 200))
        keep = rng.random(n) < rng.choice([0.02, 0.5, 0.9, 0.99, 1.0])
        if trial % 7 == 0:
            keep[: int(rng.integers(0, n + 1))] = True                     # removals only in the tail (the steady state)
        data = np.arange(n) + 1000
        store = data.copy()
        nblk = (n + B - 1) // B
        sums = np.array([keep[b * B:(b + 1) * B].sum() for b in range(nblk)])
        offs = np.concatenate([[0], np.cumsum(sums)[:-1]])
        full = np.array([min(B, n - b * B) for b in range(nblk)])
        first = next((b for b in range(nblk) if sums[b] != B), nblk)        # k_scan_block_sums: first sub-block with a removal (or a partial one)
        assert all(sums[b] == full[b] == B for b in range(first))           # everything before it stays in place
        loaded_src = np.zeros(n, bool)                                      # source entries whose value sits in some worker's registers
        loaded_src[: first * B] = True                                      # never touched: nobody writes there (checked below)
        published = np.zeros(nblk, bool)
        regs = {}
        next_ticket, workers, done = first, [None] * int(rng.integers(1, 5)), 0
        guard = 0
        while done < nblk - first:
            guard += 1
            assert guard < 100000, "schedule does not terminate"
            w = int(rng.integers(0, len(workers)))
            st = workers[w]
            if st is None:
                if next_ticket < nblk:
                    workers[w] = ["load", next_ticket]; next_ticket += 1
                continue
            phase, b = st
            lo, hi = b * B, min((b + 1) * B, n)
            if phase == "load":
                idx = [e for e in range(lo, hi) if keep[e]]
                regs[b] = [(e, store[e]) for e in idx]
                for e in idx:
                    assert store[e] == data[e], "a survivor was overwritten before its sub-block loaded it"
                loaded_src[lo:hi] = True
                published[b] = True
                st[0] = "store"
            else:
                if sums[b]:
                    s0, s1 = offs[b] // B, (offs[b] + sums[b] - 1) // B
                    deps = [s for s in range(s0, s1 + 1) if s < b]
                    assert all(s >= first for s in deps)
                    if not all(published[s] for s in deps):
                        assert all(s < b for s in deps)                      # waits only point to lower tickets
                        continue
                for k, (e, v) in enumerate(regs.pop(b)):
                    d = offs[b] + k
                    assert d <= e
                    if d != e:
                        assert loaded_src[d], "store onto a source entry that has not been loaded"
                        store[d] = v
                workers[w] = None; done += 1
        m = int(keep.sum())
        assert np.array_equal(store[:m], data[keep]), (trial, n)
