"""GPU parity tests: the CUDA path (through the C ABI) against the CPU oracle on the same
seeded synthetic inputs.  Integer / index / per-element fp32 outputs must be BIT-EXACT;
Gauss-Newton reductions (summation order differs) are checked to the tolerances written
next to each assertion.  Run on an H100: pytest -m gpu."""
from __future__ import annotations

import json
import os

import numpy as np
import pytest

from tests import oracle_lib as ol
from tests.stagewise import OracleStages, mismatch, planar_valid_equal

pytestmark = pytest.mark.gpu

W, H = 640, 480
OUT = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "gpurun_out")


class Report:
    def __init__(self, name):
        self.name, self.fail, self.log = name, [], []

    def check(self, what, ok, detail=""):
        self.log.append(f"{'ok  ' if ok else 'FAIL'} {what} {detail}")
        if not ok:
            self.fail.append(f"{what} {detail}")

    def exact(self, what, a, b):
        n, _ = mismatch(a, b)
        self.check(what, n == 0, f"mismatches={n}/{np.asarray(a).size}")

    def planar(self, what, a, b):
        ok, n = planar_valid_equal(a, b)
        self.check(what, ok, f"mismatches={n}")

    def finish(self):
        os.makedirs(OUT, exist_ok=True)
        with open(os.path.join(OUT, f"parity_{self.name}.log"), "w") as f:
            f.write("\n".join(self.log) + "\n")
        assert not self.fail, f"{len(self.fail)} parity failures (first 12): " + " | ".join(self.fail[:12])


def make_pair(**kw):
    import maskfusion_b200 as mfb
    from maskfusion_b200.synth import SynthScene
    cap = kw.pop("capacityGlobal", 1200000)
    ocfg = ol.default_config(W, H, capacityGlobal=cap, **kw)
    ccfg = mfb.default_config(W, H, capacityGlobal=cap, **kw)
    return SynthScene(W, H, n_objects=0, seed=0), OracleStages(ocfg), mfb.MaskFusion(ccfg)


def run_stagewise(name, nframes, clean_conf=None, **kw):
    sc, orc, mf = make_pair(**kw)
    rep = Report(name)
    gm = mf.getBackgroundModel()
    tick = 1
    pose_err = []
    for t in range(nframes):
        rgb, depth, *_ = sc.render(t)
        orc.set_frame(rgb, depth)
        orc.tick = tick
        fa = orc.frame_arrays()
        if t == 0:
            mf.setFrame(rgb, depth)
            rep.exact(f"[{t}] bilateral", mf.filteredDepth(), fa["depthFilt"])
            orc.init_first(); gm.initialise(tick)
            # initFirstRGB on the CUDA side happens inside processFrame; stage-wise we replicate via a hidden track-less path:
            so, sm = orc.p.surfels(0), gm.downloadMap()
            rep.check(f"[{t}] init count", so.shape[0] == sm.shape[0], f"{so.shape[0]} vs {sm.shape[0]}")
            if so.shape == sm.shape:
                rep.exact(f"[{t}] init surfels", sm, so)
        else:
            mf.setFrame(rgb, depth)
            rep.exact(f"[{t}] bilateral", mf.filteredDepth(), fa["depthFilt"])
            orc.generate_maps()
            for l in range(3):
                d, v, n = mf.frameMaps(l)
                if l > 0:
                    rep.exact(f"[{t}] depth pyr L{l}", d, fa[f"depth{l}"])
                rep.planar(f"[{t}] vmap L{l}", v, fa[f"vmap{l}"])
                rep.planar(f"[{t}] nmap L{l}", n, fa[f"nmap{l}"])
            orc.track()
            gm.performTracking()
            od = orc.odom(0)
            for l in range(3):
                v, n = gm.modelMaps(l)
                rep.planar(f"[{t}] model vmap L{l}", v, ol.arr(od.vmap_g[l], (3, H >> l, W >> l), np.float32))
                rep.planar(f"[{t}] model nmap L{l}", n, ol.arr(od.nmap_g[l], (3, H >> l, W >> l), np.float32))
            Po, Pc = orc.pose(0), gm.getPose()
            dt = float(np.linalg.norm(Po[:3, 3] - Pc[:3, 3])); dR = float(np.abs(Po[:3, :3] - Pc[:3, :3]).max())
            pose_err.append(dt)
            # fp64 sums of exact products rounded to float + the oracle's pivoted LDLT reproduced operation for operation: the tracked
            # pose is the oracle's pose BIT FOR BIT (a sum straddling a float rounding boundary has probability ~1e-7 per value)
            rep.check(f"[{t}] tracked pose", dt < 2e-5 and dR < 2e-5, f"dt={dt:.3e} dR={dR:.3e}")
            rep.check(f"[{t}] tracked pose bit-exact", np.array_equal(Po, Pc), f"dt={dt:.3e} dR={dR:.3e}")
            A, b, e = gm.trackStats()
            Ao = np.array(od.lastA).reshape(6, 6); bo = np.array(od.lastb)
            # last-iteration system: A to 1e-5 relative; b (which is ~0 at convergence) relative to |A|, not to itself
            relA = float(np.abs(A - Ao).max() / (np.abs(Ao).max() + 1e-30)); relb = float(np.abs(b - bo).max() / (np.abs(Ao).max() + 1e-30))
            rep.check(f"[{t}] last JtJ/Jtr", relA < 1e-5 and relb < 1e-5, f"relA={relA:.2e} relb={relb:.2e}")
            rep.check(f"[{t}] last JtJ/Jtr bit-exact", np.array_equal(A, Ao) and np.array_equal(b, bo), f"relA={relA:.2e} relb={relb:.2e}")
            # residual statistics of the last iteration: the counts are integers decided per pixel (a pixel may flip at a ~1e-9 pose difference)
            eo = np.array([od.lastICPError, od.lastICPCount, od.lastRGBError, od.lastRGBCount], np.float64)
            rep.check(f"[{t}] ICP count", abs(e[1] - eo[1]) <= max(3, 1e-4 * eo[1]) and eo[1] > 1000, f"{e[1]} vs {eo[1]}")
            rep.check(f"[{t}] ICP error", abs(e[0] - eo[0]) <= 1e-4 * abs(eo[0]) + 1e-12, f"{e[0]} vs {eo[0]}")
            if mf.cfg.icpWeight < 100:
                rep.check(f"[{t}] RGB correspondences", abs(e[3] - eo[3]) <= max(3, 1e-4 * eo[3]) and eo[3] > 1000, f"{e[3]} vs {eo[3]}")
                rep.check(f"[{t}] RGB error", abs(e[2] - eo[2]) <= 1e-4 * abs(eo[2]) + 1e-12, f"{e[2]} vs {eo[2]}")
            gm.debugSetPoses(Po, orc.last_pose(0))          # teacher forcing
            orc.predict_indices(); gm.predictIndices(tick)
            idx, vc, ct, nr = gm.indexMap()
            rep.exact(f"[{t}] index map ids", idx, orc.p.tex(0, "idx"))
            rep.exact(f"[{t}] index vertConf", vc, orc.p.tex(0, "vertConf"))
            rep.exact(f"[{t}] index colorTime", ct, orc.p.tex(0, "colorTime"))
            rep.exact(f"[{t}] index normRad", nr, orc.p.tex(0, "normRad"))
            orc.fuse(); gm.fuse(tick, mf.cfg.depthCutoff, 1.0)
            flag, best, meas = gm.association()
            fo, bo_, mo = orc.p.tex(0, "updateId"), orc.p.tex(0, "best"), orc.p.tex(0, "meas")
            rep.exact(f"[{t}] assoc flags", flag, fo)
            sel = fo > 0
            rep.exact(f"[{t}] assoc best", best[fo == 1], bo_[fo == 1])
            rep.exact(f"[{t}] assoc meas", meas[sel], mo[sel])
            so, sm = orc.p.surfels(0), gm.downloadMap()
            rep.check(f"[{t}] fused count", so.shape == sm.shape, f"{so.shape} vs {sm.shape}")
            if so.shape == sm.shape:
                rep.exact(f"[{t}] fused surfels", sm, so)
            orc.predict_indices(); gm.predictIndices(tick)
            rep.exact(f"[{t}] index map ids (2)", gm.indexMap()[0], orc.p.tex(0, "idx"))
            if clean_conf is not None:
                # Model::clean called with another confidence threshold than the index map was resolved with: the packed window texels
                # (whose sign bits carry `conf > threshold`) are not valid for this call, the window reads the index-map images instead
                orc.mptr(0).contents.confThreshold = clean_conf; gm.setConfidenceThreshold(clean_conf)
            orc.clean(); gm.clean(tick)
            so, sm = orc.p.surfels(0), gm.downloadMap()
            rep.check(f"[{t}] clean count", so.shape[0] == sm.shape[0], f"{so.shape[0]} vs {sm.shape[0]}")
            if so.shape == sm.shape:
                rep.exact(f"[{t}] clean surfels (ordered)", sm, so)
        orc.predict(); gm.combinedPredict(tick, tick)
        im, vc, nr, tt = gm.prediction()
        rep.exact(f"[{t}] splat image", im, orc.p.tex(0, "splatImage"))
        rep.exact(f"[{t}] splat vertex", vc, orc.p.tex(0, "splatVertex"))
        rep.exact(f"[{t}] splat normal", nr, orc.p.tex(0, "splatNormal"))
        rep.exact(f"[{t}] splat time", tt, orc.p.tex(0, "splatTime"))
        fim, fv, fn = gm.fillIn()
        rep.exact(f"[{t}] fill image", fim, orc.p.tex(0, "fillImage"))
        rep.exact(f"[{t}] fill vertex", fv, orc.p.tex(0, "fillVertex"))
        rep.exact(f"[{t}] fill normal", fn, orc.p.tex(0, "fillNormal"))
        if t == 0:
            # CUDA-side initFirstRGB equivalent for the stage-wise driver: run a real processFrame on a twin? Not needed:
            # so3 is exercised by the free-running sequence test; stage-wise runs use so3 only after frame 0 via processFrame state.
            pass
        tick += 1
    rep.log.append("pose errors vs oracle (m): " + json.dumps(pose_err))
    mf.close()
    rep.finish()


def test_stagewise_icp_only():
    """-static, ICP-only tracking (icpWeight=100 => rgb=false, RGBDOdometry.cpp:236-237), no SO3"""
    run_stagewise("stagewise_icp", 6, icpWeight=100.0, so3=0)


def test_stagewise_clean_with_other_threshold():
    """the fallback of the clean window (three index-map images instead of the packed 16-byte texels): confidence threshold changed between
    Model::predictIndices and Model::clean"""
    run_stagewise("stagewise_clean_conf", 4, clean_conf=3.0, icpWeight=100.0, so3=0)


def test_stagewise_rgbd():
    """-static, GUI-default ICP+RGB weighting (icpWeight=20), no SO3 (needs initFirstRGB state: see sequence test)"""
    run_stagewise("stagewise_rgbd", 4, icpWeight=20.0, so3=0)


def _run_sequences(n, **kw):
    import maskfusion_b200 as mfb
    from maskfusion_b200.synth import SynthScene
    sc = SynthScene(W, H, n_objects=0, seed=1)
    cap = 1500000
    orc = ol.OraclePipeline(ol.default_config(W, H, capacityGlobal=cap, **kw))
    mf = mfb.MaskFusion(mfb.default_config(W, H, capacityGlobal=cap, **kw))
    agree = []
    for t in range(n):
        rgb, depth, *_ = sc.render(t)
        orc.process_frame(rgb, depth, t * 33333)
        mf.processFrame(rgb, depth, t * 33333)
    mf.sync()
    lo = np.array([orc.model(0).log[i] for i in range(orc.model(0).nlog * 8)]).reshape(-1, 8)
    lc = mf.getBackgroundModel().poseLog()
    # MaskFusion::exportPoses: the file holds the same log, seconds first, 6 decimals
    import tempfile
    with tempfile.TemporaryDirectory() as d:
        assert mf.exportPoses(d + "/") == 1
        txt = np.loadtxt(os.path.join(d, "poses-0.txt")).reshape(-1, 8)
    assert txt.shape == lc.shape and np.allclose(txt[:, 0], lc[:, 0] * 1e-6, atol=1e-6) and np.allclose(txt[:, 1:], lc[:, 1:], atol=1e-6)
    counts = (orc.count(0), mf.getBackgroundModel().lastCount())
    # index-map agreement on the final state (free-running, no teacher forcing): the oracle's last predictIndices ran BEFORE its
    # clean, so both sides re-project their final (cleaned) stores with the final pose and time
    mf.getBackgroundModel().predictIndices(mf.getTick() - 1)
    idx_c = mf.getBackgroundModel().indexMap()[0]
    so, sm = orc.surfels(0), mf.getBackgroundModel().downloadMap()
    final = {"surfels_equal": so.shape == sm.shape and bool(np.array_equal(so.view(np.uint32), sm.view(np.uint32))),
             "pose_equal": bool(np.array_equal(orc.pose(0), mf.getBackgroundModel().getPose()))}
    mf.close()
    return lo, lc, counts, idx_c, orc, final


def test_sequence_ate_icp():
    """free-running 16-frame replay, ICP only: per-frame translation within 1 mm ATE-RMSE of the oracle"""
    lo, lc, counts, idx_c, orc, final = _run_sequences(16, icpWeight=100.0, so3=0)
    assert lo.shape == lc.shape
    assert np.array_equal(lo[:, 0], lc[:, 0])
    ate = float(np.sqrt(np.mean(np.sum((lo[:, 1:4] - lc[:, 1:4]) ** 2, axis=1))))
    assert ate < 1e-3, f"ATE-RMSE {ate*1e3:.4f} mm"
    assert abs(counts[0] - counts[1]) <= max(50, counts[0] // 2000), counts
    # bit-identical free-running trajectory => bit-identical stores (VERDICT r1: assert on the final state, not only on the poses)
    assert np.array_equal(lo, lc), f"pose logs differ: max {np.abs(lo - lc).max():.3e}"
    assert counts[0] == counts[1] and final["surfels_equal"] and final["pose_equal"], (counts, final)


def test_sequence_ate_rgbd_so3():
    """free-running 12-frame replay with the GUI defaults (ICP+RGB, SO3 pre-alignment)"""
    lo, lc, counts, idx_c, orc, final = _run_sequences(12)
    ate = float(np.sqrt(np.mean(np.sum((lo[:, 1:4] - lc[:, 1:4]) ** 2, axis=1))))
    assert ate < 1e-3, f"ATE-RMSE {ate*1e3:.4f} mm"
    assert np.array_equal(lo, lc), f"pose logs differ: max {np.abs(lo - lc).max():.3e}"
    assert counts[0] == counts[1] and final["surfels_equal"] and final["pose_equal"], (counts, final)


def test_bench_state_matches_oracle():
    """The benchmarked state (VERDICT r1): capacity 2176^2, the background store pre-populated to ~4.6 M surfels exactly as bench.py does,
    GUI defaults (ICP+RGB w=20, SO3), free running.  After three frames: pose logs, surfel stores (bit patterns), the index map of the last
    predictIndices (the one that rides inside Model::clean) and the splat prediction equal the oracle's."""
    import ctypes as C
    import maskfusion_b200 as mfb
    from maskfusion_b200.synth import SynthScene, dense_room_surfels
    cap, prepop = 2176 * 2176, 4_300_000
    sc = SynthScene(W, H, n_objects=0, seed=0)
    orc = ol.OraclePipeline(ol.default_config(W, H, capacityGlobal=cap))
    mf = mfb.MaskFusion(mfb.default_config(W, H, capacityGlobal=cap))
    rgb, depth, *_ = sc.render(0)
    orc.process_frame(rgb, depth, 0)
    mf.processFrame(rgb, depth, 0)
    gm = mf.getBackgroundModel()
    cur = gm.downloadMap()
    assert np.array_equal(cur.view(np.uint32), orc.surfels(0).view(np.uint32))
    room = dense_room_surfels(sc, prepop, time=1, conf=20.0)
    Tinv = np.linalg.inv(sc.camera_pose(0))
    room[:, 0:3] = (room[:, 0:3].astype(np.float64) @ Tinv[:3, :3].T + Tinv[:3, 3]).astype(np.float32)
    room[:, 8:11] = (room[:, 8:11].astype(np.float64) @ Tinv[:3, :3].T).astype(np.float32)
    allv = np.ascontiguousarray(np.concatenate([cur, room], 0))
    gm.uploadMap(allv)
    m = orc.L.orc_mf_model(orc.h, 0)
    C.memmove(m.contents.surf[m.contents.target], allv.ctypes.data, allv.nbytes)
    m.contents.count = allv.shape[0]
    for t in range(1, 4):
        rgb, depth, *_ = sc.render(t)
        orc.process_frame(rgb, depth, t * 33333)
        mf.processFrame(rgb, depth, t * 33333)
    mf.sync()
    lo = np.array([orc.model(0).log[i] for i in range(orc.model(0).nlog * 8)]).reshape(-1, 8)
    lc = gm.poseLog()
    assert np.array_equal(lo, lc), f"pose logs differ: max {np.abs(lo - lc).max():.3e}"
    assert orc.count(0) == gm.lastCount() and orc.count(0) > 4_400_000, (orc.count(0), gm.lastCount())
    so, sm = orc.surfels(0), gm.downloadMap()
    assert np.array_equal(so.view(np.uint32), sm.view(np.uint32)), int((so.view(np.uint32) != sm.view(np.uint32)).any(axis=1).sum())
    idx_c, vc_c, ct_c, nr_c = gm.indexMap()
    assert np.array_equal(idx_c, orc.tex(0, "idx")), int((idx_c != orc.tex(0, "idx")).sum())
    assert np.array_equal(vc_c.view(np.uint32), orc.tex(0, "vertConf").view(np.uint32))
    im, pv, pn, tt = gm.prediction()
    assert np.array_equal(pv.view(np.uint32), orc.tex(0, "splatVertex").view(np.uint32))
    assert np.array_equal(im, orc.tex(0, "splatImage")) and np.array_equal(tt, orc.tex(0, "splatTime"))
    mf.close()


def test_icp_step_matches_oracle():
    """icpStep (reduce.cu:446-525) at a fixed pose: 29 sums within 1e-4 relative of the double-precision oracle"""
    import ctypes as C
    sc, orc, mf = make_pair(icpWeight=100.0, so3=0)
    gm = mf.getBackgroundModel()
    for t in range(2):
        rgb, depth, *_ = sc.render(t)
        orc.p.process_frame(rgb, depth, t)
        mf.processFrame(rgb, depth, t)
    rgb, depth, *_ = sc.render(2)
    orc.set_frame(rgb, depth); orc.generate_maps(); orc.track()
    mf.setFrame(rgb, depth); gm.performTracking()
    od = orc.odom(0)
    L = orc.L
    R = np.eye(3, dtype=np.float32); tv = np.zeros(3, np.float32)
    P = orc.last_pose(0)
    for l in range(3):
        w, h = W >> l, H >> l
        fa = orc.frame_arrays()
        Rpi = np.linalg.inv(P[:3, :3].astype(np.float64)).astype(np.float32)
        Rc = P[:3, :3].copy(); tc = P[:3, 3].copy()
        out = np.zeros(29)
        cam = ol.cam(528.0 / (1 << l), 528.0 / (1 << l), 320.0 / (1 << l), 240.0 / (1 << l))
        L.orc_icp_step(ol.ptr(np.ascontiguousarray(Rc)), ol.ptr(np.ascontiguousarray(tc)), ol.ptr(fa[f"vmap{l}"]), ol.ptr(fa[f"nmap{l}"]),
                       ol.ptr(np.ascontiguousarray(Rpi)), ol.ptr(np.ascontiguousarray(P[:3, 3].copy())), cam,
                       od.vmap_g[l], od.nmap_g[l], C.c_float(0.1), C.c_float(np.float32(np.sin(20.0 * 3.14159254 / 180.0))), w, h, ol.ptr(out))
        gm.debugSetPoses(P, P)
        got = gm.icpStep(l, Rc, tc).astype(np.float64)
        assert abs(got[28] - out[28]) <= 2, (l, got[28], out[28])   # inlier count (Rprev^-1 is formed differently in this test: ulp-level gate differences)
        scale = np.abs(out[:27]).max()
        assert np.abs(got[:28] - out[:28]).max() <= 1e-4 * max(scale, 1.0), (l, np.abs(got - out).max(), scale)
    mf.close()


def test_edge_map_matches_oracle():
    """geometric edge-ness + threshold + invert (segmentation.cu:122-177,257-269) bit-exact"""
    import ctypes as C
    sc, orc, mf = make_pair(icpWeight=100.0, so3=0)
    rgb, depth, *_ = sc.render(3)
    orc.set_frame(rgb, depth); orc.generate_maps()
    mf.setFrame(rgb, depth)
    e, b = mf.edgeMap()
    fa = orc.frame_arrays()
    eo = np.zeros((H, W), np.float32); bo = np.zeros((H, W), np.uint8); inv = np.zeros((H, W), np.uint8)
    orc.L.orc_geometric_edges(ol.ptr(fa["vmap0"]), ol.ptr(fa["nmap0"]), W, H, C.c_float(150.0), C.c_float(2.8), ol.ptr(eo))
    orc.L.orc_threshold(ol.ptr(eo), W * H, C.c_float(0.3), ol.ptr(bo))
    orc.L.orc_invert(ol.ptr(bo), W * H, ol.ptr(inv))
    assert mismatch(e, eo)[0] == 0
    assert np.array_equal(b, inv)
    mf.close()


def test_process_frame_error_behaviour():
    """argument checks mirror the asserts of MaskFusion::processFrame (MaskFusion.cpp:201-203)"""
    import maskfusion_b200 as mfb
    mf = mfb.MaskFusion(mfb.default_config(W, H, capacityGlobal=400000))
    with pytest.raises(mfb.MFError):
        mf.processFrame(np.zeros((H, W, 3), np.uint8), np.zeros((H, W), np.float64))
    with pytest.raises(mfb.MFError):
        mf.processFrame(np.zeros((H, W, 3), np.uint8), np.zeros((H, W), np.float32), timestamp=-1)
    mf.close()


def test_sequence_720p_matches_oracle():
    """BASELINE configs[4] resolution (1280x720, fx=fy=792): free-running GUI-default replay against the oracle -- the pyramid,
    tracker (12+ pixel rounds per thread, correspondences in 49 KB of dynamic shared memory), index map and clean paths at the
    largest size the configs name; per-frame translation within 1 mm, surfel counts equal, final index map identical"""
    import maskfusion_b200 as mfb
    from maskfusion_b200.synth import SynthScene
    W2, H2 = 1280, 720
    sc = SynthScene(W2, H2, n_objects=0, seed=2)
    kw = dict(capacityGlobal=2200000, fx=792.0, fy=792.0, cx=640.0, cy=360.0)       # the "-cal" intrinsics of SURVEY 8(d)
    orc = ol.OraclePipeline(ol.default_config(W2, H2, **kw))
    mf = mfb.MaskFusion(mfb.default_config(W2, H2, **kw))
    for t in range(5):
        rgb, depth, *_ = sc.render(t)
        orc.process_frame(rgb, depth, t * 33333)
        mf.processFrame(rgb, depth, t * 33333)
        dp = float(np.abs(orc.pose(0) - mf.getBackgroundModel().getPose()).max())
        assert dp < 2e-5, (t, dp)
        co, cc = orc.count(0), mf.getBackgroundModel().lastCount()
        assert abs(co - cc) <= max(30, co // 2000), (t, co, cc)
    lo = np.array([orc.model(0).log[i] for i in range(orc.model(0).nlog * 8)]).reshape(-1, 8)
    lc = mf.getBackgroundModel().poseLog()
    ate = float(np.sqrt(np.mean(np.sum((lo[:, 1:4] - lc[:, 1:4]) ** 2, axis=1))))
    assert ate < 1e-3, f"ATE-RMSE {ate*1e3:.4f} mm"
    mf.close()


def test_degenerate_frames_match_oracle():
    """edge cases of the inputs, free-running against the oracle: an all-zero depth frame (no vertex, no correspondence: singular
    normal equations, Eigen's zero-pivot convention => no motion), a frame with 60 % holes, and a surfel store that is full
    (capacity == first frame: every later insertion is clamped exactly like the reference's fixed-size VBO)"""
    import maskfusion_b200 as mfb
    from maskfusion_b200.synth import SynthScene
    sc = SynthScene(W, H, n_objects=0, seed=4)
    kw = dict(capacityGlobal=307200, icpWeight=100.0, so3=0)
    orc = ol.OraclePipeline(ol.default_config(W, H, **kw))
    mf = mfb.MaskFusion(mfb.default_config(W, H, **kw))
    rng = np.random.default_rng(0)
    for t in range(6):
        rgb, depth, *_ = sc.render(t)
        if t == 2:
            depth = np.zeros_like(depth)
        if t == 4:
            depth = depth.copy(); depth[rng.random(depth.shape) < 0.6] = 0
        orc.process_frame(rgb, depth, t * 33333)
        mf.processFrame(rgb, depth, t * 33333)
        Po, Pc = orc.pose(0), mf.getBackgroundModel().getPose()
        assert np.all(np.isfinite(Pc)), t
        assert float(np.abs(Po - Pc).max()) < 2e-5, (t, float(np.abs(Po - Pc).max()))
        co, cc = orc.count(0), mf.getBackgroundModel().lastCount()
        assert cc <= 307200 and abs(co - cc) <= max(30, co // 2000), (t, co, cc)
    mf.close()
