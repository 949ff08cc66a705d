"""GPU parity of the multi-model schedule (MaskFusion.cpp:287-375): global model-ID projection,
geometric edge segmentation + the (GPU) connected-component / voting tail, model spawn, per-object
fusion -- free-running CUDA pipeline against the free-running CPU oracle on a synthetic scene with
three objects and instance masks (the "-maskdir" mode of the reference: masks are inputs)."""
from __future__ import annotations

import ctypes as C
import json
import os

import numpy as np
import pytest

from tests import oracle_lib as ol

pytestmark = pytest.mark.gpu
W, H = 640, 480
OUT = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "gpurun_out")


class MFS(C.Structure):
    _fields_ = [("cfg", ol.Config), ("cam", ol.Cam), ("tick", C.c_int), ("rgb", ol.u8p), ("depthRaw", ol.f32p), ("depthFilt", ol.f32p),
                ("mask", ol.u8p), ("depthPyr", ol.f32p * 3), ("maskPyr", ol.u8p * 3), ("vmap", ol.f32p * 3), ("nmap", ol.f32p * 3),
                ("nmodels", C.c_int), ("models", C.c_void_p * 256), ("nextID", C.c_uint8), ("spawnOffset", C.c_int),
                ("projKeys", C.c_void_p), ("projectedIDs", ol.u8p), ("fullSeg", ol.u8p)]


def run(nframes, track_all, tag="", n_objects=3, layout="room", size=None, **over):
    import maskfusion_b200 as mfb
    from maskfusion_b200.synth import SynthScene
    kw = dict(capacityGlobal=1000000, capacityObject=200000, enableMultipleModels=1, icpWeight=100.0, so3=0, trackAllModels=int(track_all))
    kw.update(over)
    W, H = size or (640, 480)
    sc = SynthScene(W, H, n_objects=n_objects, seed=0, layout=layout)
    orc = ol.OraclePipeline(ol.default_config(W, H, **kw))
    L = orc.L
    L.orc_mf_process_frame_ex.argtypes = [C.c_void_p] * 3 + [C.c_int64, C.c_void_p, C.c_void_p, C.c_int]
    mf = mfb.MaskFusion(mfb.default_config(W, H, **kw))
    cls = np.array([0] + [o.class_id for o in sc.objects], np.int32)
    log = []
    for t in range(nframes):
        rgb, depth, mask, *_ = sc.render(t)
        mask = np.ascontiguousarray(mask)
        L.orc_mf_process_frame_ex(orc.h, ol.ptr(np.ascontiguousarray(rgb)), ol.ptr(np.ascontiguousarray(depth)), t * 33333, ol.ptr(mask), ol.ptr(cls), len(cls))
        mf.processFrame(rgb, depth, t * 33333, mask=mask, classIDs=cls)
        s = C.cast(orc.h, C.POINTER(MFS)).contents
        seg_c, proj_c = mf.segmentation()
        seg_o = ol.arr(s.mask, (H, W), np.uint8); proj_o = ol.arr(s.projectedIDs, (H, W), np.uint8)
        models_c = mf.getModels()
        rec = {"t": t, "n_o": int(s.nmodels), "n_c": len(models_c),
               "seg_diff": int((seg_c != seg_o).sum()), "proj_diff": int((proj_c != proj_o).sum()),
               "ids_o": [int(orc.model(i).id) for i in range(s.nmodels)], "ids_c": [m.getID() for m in models_c],
               "cls_o": [int(orc.model(i).classID) for i in range(s.nmodels)], "cls_c": [m.getClassID() for m in models_c],
               "cnt_o": [int(orc.count(i)) for i in range(s.nmodels)], "cnt_c": [m.lastCount() for m in models_c]}
        if rec["n_o"] == rec["n_c"]:
            rec["dpose"] = [float(np.abs(orc.pose(i) - models_c[i].getPose()).max()) for i in range(rec["n_o"])]
        rec["pose_o"] = [orc.pose(i).tolist() for i in range(s.nmodels)]
        log.append(rec)
    # exported trajectories (MaskFusion.cpp:577-592: background pose, object poses as globalPose * objPose^-1), both sides
    n_final = int(C.cast(orc.h, C.POINTER(MFS)).contents.nmodels)
    traj = {"oracle": [np.array([orc.model(i).log[k] for k in range(orc.model(i).nlog * 8)]).reshape(-1, 8) for i in range(n_final)],
            "cuda": [m.poseLog() for m in mf.getModels()]}
    for r in log:
        r["traj"] = None
    log[-1]["traj"] = traj
    mf.close()
    os.makedirs(OUT, exist_ok=True)
    with open(os.path.join(OUT, f"multi_trackall{int(track_all)}_w{int(kw['icpWeight'])}{tag}.json"), "w") as f:
        json.dump([{k: v for k, v in r.items() if k != "traj"} for r in log], f)
    return log


def ate_rmse(traj):
    """per-model ATE-RMSE (translation, entries matched by timestamp, no alignment: both runs start at identity) in metres"""
    out = []
    for lo, lc in zip(traj["oracle"], traj["cuda"]):
        to = {int(r[0]): r[1:4] for r in lo}; tc = {int(r[0]): r[1:4] for r in lc}
        common = sorted(set(to) & set(tc))
        assert len(common) >= max(1, min(len(to), len(tc)) - 1), (len(to), len(tc), len(common))
        d = np.array([to[k] - tc[k] for k in common])
        out.append(float(np.sqrt(np.mean(np.sum(d * d, axis=1)))))
    return out


def check_exact(log, min_models):
    """fp64 sums + the oracle's solver reproduced operation for operation: EVERY model's pose, the segmentation, the projected-ID image
    and the surfel counts equal the oracle's on every frame (tracked objects included), hence ATE-RMSE = 0 <= 1 mm"""
    assert max(r["n_o"] for r in log) >= min_models, "oracle never spawned enough object models"
    for r in log:
        rec = {k: v for k, v in r.items() if k not in ("pose_o", "traj")}
        assert r["n_o"] == r["n_c"] and r["ids_o"] == r["ids_c"] and r["cls_o"] == r["cls_c"], rec
        assert max(r["dpose"]) == 0.0, rec
        assert r["seg_diff"] == 0 and r["proj_diff"] == 0, rec
        assert r["cnt_o"] == r["cnt_c"], rec
    ate = ate_rmse(log[-1]["traj"])
    assert max(ate) <= 1e-3, ate
    return ate


def oracle_poses(nframes, eps, **over):
    """free-running oracle alone, every reduced sum of the tracker scaled by (1 + eps*u), |u| <= 1 (orc_debug_set_sum_perturb):
    how far rounding-size noise in the normal equations moves each model's pose"""
    from maskfusion_b200.synth import SynthScene
    kw = dict(capacityGlobal=1000000, capacityObject=200000, enableMultipleModels=1, icpWeight=100.0, so3=0, trackAllModels=1)
    kw.update(over)
    sc = SynthScene(W, H, n_objects=3, seed=0)
    orc = ol.OraclePipeline(ol.default_config(W, H, **kw))
    L = orc.L
    L.orc_debug_set_sum_perturb.argtypes = [C.c_double]
    L.orc_mf_process_frame_ex.argtypes = [C.c_void_p] * 3 + [C.c_int64, C.c_void_p, C.c_void_p, C.c_int]
    cls = np.array([0] + [o.class_id for o in sc.objects], np.int32)
    out = []
    L.orc_debug_set_sum_perturb(eps)
    try:
        for t in range(nframes):
            rgb, depth, mask, *_ = sc.render(t)
            mask = np.ascontiguousarray(mask)
            L.orc_mf_process_frame_ex(orc.h, ol.ptr(np.ascontiguousarray(rgb)), ol.ptr(np.ascontiguousarray(depth)), t * 33333, ol.ptr(mask), ol.ptr(cls), len(cls))
            n = C.cast(orc.h, C.POINTER(MFS)).contents.nmodels
            out.append([orc.pose(i).copy() for i in range(n)])
    finally:
        L.orc_debug_set_sum_perturb(0.0)
    return out


def check(log, min_models, envelope=None):
    """envelope[t][i]: pose distance the oracle itself moves under fp32-rounding-size noise (tracked object models only)"""
    assert max(r["n_o"] for r in log) >= min_models, "oracle never spawned an object model"
    worst = {}
    for r in log:
        assert r["n_o"] == r["n_c"], r["t"]
        assert r["ids_o"] == r["ids_c"] and r["cls_o"] == r["cls_c"], r["t"]
        rec = {k: v for k, v in r.items() if k != "pose_o"}
        if envelope is None:
            # bit-exact kernels + poses that agree to ~1e-8: the images agree except (rarely) at a pixel whose depth test flips
            assert r["proj_diff"] <= 20, rec
            assert r["seg_diff"] <= 200, rec
            for a, b in zip(r["cnt_o"], r["cnt_c"]):
                assert abs(a - b) <= max(30, a // 500), rec
            assert max(r["dpose"]) < 2e-5, rec
            continue
        # tracked objects: a freshly spawned object model (3-5k surfels) gives near-singular normal equations; noise of the size of
        # one fp32 rounding in the reduced sums moves the ORACLE's own object poses by 1e-4 .. 1e-2 (envelope), the background by < 1e-7.
        # The CUDA path must stay inside that envelope (x10, running maximum) and bit-for-bit comparable where the problem is well posed.
        assert r["dpose"][0] < 2e-5, rec                                     # background: well conditioned
        assert abs(r["cnt_o"][0] - r["cnt_c"][0]) <= max(30, r["cnt_o"][0] // 500), rec
        for i in range(1, r["n_o"]):
            e = envelope[r["t"]][i] if i < len(envelope[r["t"]]) else 0.0
            worst[i] = max(worst.get(i, 0.0), e)
            assert r["dpose"][i] <= max(2e-5, 10.0 * worst[i]), (rec, worst)
            assert r["dpose"][i] < 5e-2, rec                                  # and never a gross failure
            assert abs(r["cnt_o"][i] - r["cnt_c"][i]) <= max(60, r["cnt_o"][i] // 20), rec
        assert r["seg_diff"] <= 3000 and r["proj_diff"] <= 3000, rec          # object silhouettes move by a pixel at most


def test_multi_model_static_objects():
    """GUI default: objects are spawned from the masks and follow the camera (trackAllModels=false, N13)"""
    log = run(26, track_all=False)
    check(log, 2)
    check_exact(log, 2)


def test_multi_model_tracked_objects():
    """trackAllModels=true, ICP only: every object model runs its own ICP, batched with the background in one launch sequence.
    The near-singular ICP system of a freshly spawned 3k-surfel object makes its first step jump > 0.2 m, so the reference rule
    (MaskFusion.cpp:268-272) removes it on the next frame -- the lifecycle (spawn, inactivate) must match the oracle exactly."""
    log = run(27, track_all=True)
    check(log, 2)
    check_exact(log, 2)
    assert log[-1]["n_c"] == 1


def test_multi_model_three_tracked_objects():
    """BASELINE configs[2] shape: three objects, each tracked with ICP + photometric term (GUI default icpWeight=20) in the
    batched persistent tracking kernel; a spawn every 6 frames so that all three exist after 18 frames and are tracked for 6 more"""
    over = dict(icpWeight=20.0, modelSpawnOffset=6)
    log = run(24, track_all=True, **over)
    assert log[-1]["n_c"] == 4
    try:
        check_exact(log, 4)
    except AssertionError:
        # diagnostic only (round-1 envelope probe): how far rounding-size noise moves the oracle's own poses on this sequence
        ref = [[np.array(p, np.float32) for p in r["pose_o"]] for r in log]
        per = oracle_poses(24, 1e-7, **over)
        envelope = [[float(np.abs(a - b).max()) for a, b in zip(pa, pb)] for pa, pb in zip(ref, per)]
        with open(os.path.join(OUT, "multi_envelope_w20.json"), "w") as f:
            json.dump({"envelope": envelope, "cuda_vs_oracle": [r.get("dpose") for r in log]}, f)
        raise


def test_table_scene_eight_tracked_objects():
    """BASELINE configs[3] scene (SURVEY 8d): eight objects of 0.2-0.4 m on a table / shelf at 1-2 m (17-23 k pixels each), static for
    30 frames and then moving <= 8 mm per frame, each tracked with ICP + photometric term next to the background.  Every pose of every
    model on every frame, the segmentation and ID images and the surfel counts must equal the oracle's; per-object ATE-RMSE of the
    exported trajectories (MaskFusion.cpp:577-592) <= 1 mm follows (it is 0).  MF_LONG=1 runs the 300-frame sequence of SURVEY 8(d)."""
    n = 300 if os.environ.get("MF_LONG") == "1" else 64
    log = run(n, track_all=True, tag=f"_table8_{n}", n_objects=8, layout="table", icpWeight=20.0, modelSpawnOffset=3)
    assert log[-1]["n_c"] == 9, log[-1]["n_c"]
    ate = check_exact(log, 9)
    with open(os.path.join(OUT, f"ate_table8_{n}.json"), "w") as f:
        json.dump({"frames": n, "ate_rmse_m": ate, "models": log[-1]["n_c"]}, f)


def test_table_scene_720p_sixteen_objects():
    """BASELINE configs[4] shape on one GPU: 1280x720 (the -cal intrinsics 792/792/640/360), sixteen objects on three rows, every model
    tracked; a spawn every frame at most (the oracle holds 12 models from frame 38 on).  Same exactness contract as the VGA scene."""
    log = run(40, track_all=True, tag="_table16_720p", n_objects=16, layout="table", size=(1280, 720), icpWeight=20.0, modelSpawnOffset=1,
              fx=792.0, fy=792.0, cx=640.0, cy=360.0, capacityGlobal=2200000, capacityObject=262144)
    assert log[-1]["n_c"] >= 12, log[-1]["n_c"]          # the partly occluded back-row objects stay below minRelSizeNew (1.5 % of the image)
    check_exact(log, 12)
