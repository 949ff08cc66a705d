"""The on-GPU Mask R-CNN detector on the frame path (mf_attach_detector / MaskFusion.attachDetector): segmentation frames that the caller
gives no mask take the detector's id image and class list (MfSegmentation.cpp:128-131, MaskRCNN.cpp:98-151).

Checked on seeded synthetic scenes with seeded network weights at 640x480:
  - the hand-off delivers exactly the detector's output, only on the frames the every_k rule selects;
  - a detector-driven context computes the same bits as a context fed the recorded masks as inputs (host and device inputs);
  - the CPU oracle fed the detector-made masks agrees with the detector-driven context on every frame, and objects are spawned from them;
  - a caller's mask takes precedence over the detector; the refusals, the export-error flag and the lifecycle."""
from __future__ import annotations

import ctypes as C

import numpy as np
import pytest

from tests import oracle_lib as ol

pytestmark = pytest.mark.gpu
W, H = 640, 480
N_FRAMES = 14
# the multi-model settings of tests/test_gpu_multi.py (exact oracle parity: ICP only, no SO3 pre-alignment).  Spawning from the detector's
# masks: a mask must cover 65 % of a geometric component to claim it, and the seeded network's boxes are not the scene's objects, so the
# claimed areas are small: minRelSizeNew = 0.002 (614 pixels) instead of 1.5 %, and a spawn may follow 2 frames after the last one.
KW = dict(capacityGlobal=1000000, capacityObject=200000, enableMultipleModels=1, icpWeight=100.0, so3=0, trackAllModels=0,
          modelSpawnOffset=2, minRelSizeNew=0.002)


@pytest.fixture(scope="module")
def frames():
    """the BASELINE configs[2] scene: table layout, three objects, seed 0"""
    from maskfusion_b200.synth import SynthScene
    sc = SynthScene(W, H, n_objects=3, seed=0, layout="table")
    out = []
    for t in range(N_FRAMES):
        rgb, depth, mask, *_ = sc.render(t)
        out.append((np.ascontiguousarray(rgb), np.ascontiguousarray(depth), np.ascontiguousarray(mask)))
    return out, np.array([0] + [o.class_id for o in sc.objects], np.int32)


@pytest.fixture(scope="module")
def nets():
    """S -> Detector (seeded backbone 7, RPN 11, heads 13: the weights of tests/test_gpu_heads.py) on a stream of its own"""
    import torch
    import maskfusion_b200 as mfb
    made = {}

    def get(S):
        if S not in made:
            st = torch.cuda.Stream()
            bb = mfb.Backbone(S, seed=7, stream=st.cuda_stream)
            rpn = mfb.RegionProposals(bb, seed=11)
            det = mfb.Detector(rpn, seed=13)
            made[S] = (st, bb, rpn, det)
        det = made[S][3]
        det.set_export()
        return det

    yield get
    for st, bb, rpn, det in made.values():
        det.close(); rpn.close(); bb.close()


def _ctx(**over):
    import maskfusion_b200 as mfb
    kw = dict(KW); kw.update(over)
    return mfb.MaskFusion(mfb.default_config(W, H, **kw))


def _state(mf):
    """everything a frame decides that the tests compare: models (ids, classes, poses as bits, surfel counts), segmentation, projected ids"""
    ms = mf.getModels()
    seg, proj = mf.segmentation()
    return {"ids": [m.getID() for m in ms], "cls": [m.getClassID() for m in ms],
            "poses": [np.asarray(m.getPose(), np.float32).view(np.uint32).copy() for m in ms], "counts": [m.lastCount() for m in ms],
            "seg": seg, "proj": proj}


def _same_state(a, b, t):
    assert a["ids"] == b["ids"] and a["cls"] == b["cls"], (t, a["ids"], b["ids"], a["cls"], b["cls"])
    assert all(np.array_equal(x, y) for x, y in zip(a["poses"], b["poses"])), t
    assert a["counts"] == b["counts"], (t, a["counts"], b["counts"])
    assert np.array_equal(a["seg"], b["seg"]) and np.array_equal(a["proj"], b["proj"]), t


def _stores(mf):
    return [np.ascontiguousarray(m.downloadMap()).view(np.uint32).copy() for m in mf.getModels()]


def _detect_runs(tick, every_k):
    return tick > 1 and tick % every_k == 0


def _run_pair(det, fr, cls, every_k, on_device, explicit=None):
    """context A (detector attached) and context B (no detector, fed A's recorded masks; mask=None where A carried none) frame by frame.
    explicit: {frame: True} -> that frame gets the scene's own mask + classes in BOTH contexts.  Returns the per-frame hand-off records."""
    import torch
    A, B = _ctx(), _ctx()
    A.attachDetector(det, every_k)
    dev = [(torch.from_numpy(r).cuda(), torch.from_numpy(d).cuda(), torch.from_numpy(m).cuda()) for r, d, m in fr] if on_device else None
    torch.cuda.synchronize()
    recs, keep = [], []                                     # B's device masks stay alive until the contexts are done with them
    try:
        for t, (rgb, depth, smask) in enumerate(fr):
            tick = A.getTick()
            before = det.idImage()
            given = bool(explicit and explicit.get(t))
            if given:
                A.setFrameClasses(cls)
            if on_device:
                A.processFramePtr(dev[t][0].data_ptr(), dev[t][1].data_ptr(), t * 33333, True, mask_ptr=dev[t][2].data_ptr() if given else 0)
            else:
                A.processFrame(rgb, depth, t * 33333, mask=smask if given else None)
            mask, ids = A.frameMasks()
            img, ecls, _ = det.idImage()
            ran = _detect_runs(tick, every_k) and not given
            recs.append({"t": t, "ran": ran, "given": given, "mask": mask, "ids": ids, "img": img, "ecls": ecls, "before": before})
            # B: the same frame with A's masks as inputs
            if ids:
                B.setFrameClasses(np.array(ids, np.int32))
                if on_device:
                    md = torch.from_numpy(mask).cuda(); torch.cuda.synchronize(); keep.append(md)
                    B.processFramePtr(dev[t][0].data_ptr(), dev[t][1].data_ptr(), t * 33333, True, mask_ptr=md.data_ptr())
                else:
                    B.processFrame(rgb, depth, t * 33333, mask=mask)
            elif on_device:
                B.processFramePtr(dev[t][0].data_ptr(), dev[t][1].data_ptr(), t * 33333, True)
            else:
                B.processFrame(rgb, depth, t * 33333)
            A.sync(); B.sync()                                  # both apply what the frame decided (a spawn) before the read-back
            _same_state(_state(A), _state(B), t)
        sa, sb = _stores(A), _stores(B)
        assert len(sa) == len(sb) and all(np.array_equal(x, y) for x, y in zip(sa, sb))
        recs[-1]["models"] = len(sa)
    finally:
        A.attachDetector(None)
        A.close(); B.close()
    return recs


def _check_handoff(recs):
    for r in recs:
        if r["ran"]:
            assert np.array_equal(r["mask"], r["img"]), (r["t"], int((r["mask"] != r["img"]).sum()))
            assert r["ids"] == [0] + r["ecls"], (r["t"], r["ids"], r["ecls"])
        elif not r["given"]:
            assert r["ids"] == [] and not r["mask"].any(), (r["t"], r["ids"])


@pytest.mark.parametrize("every_k", [1, 2])
@pytest.mark.parametrize("S", [256, 1024])
def test_handoff_is_the_detector_output(nets, frames, S, every_k):
    """after every frame: frameMasks() is the detector's id image and [0] + its class ids on the frames the rule selects, nothing on the
    others (frame 1, skipped ticks); the id image equals execute() on the same RGB (the frame's RGBA copy is what the detector saw)"""
    det = nets(S)
    fr, _ = frames
    mf = _ctx()
    mf.attachDetector(det, every_k)
    ran = 0
    try:
        for t, (rgb, depth, _) in enumerate(fr):
            tick = mf.getTick()
            mf.processFrame(rgb, depth, t * 33333)
            mask, ids = mf.frameMasks()
            img, ecls, _ = det.idImage()
            if _detect_runs(tick, every_k):
                ran += 1
                assert np.array_equal(mask, img), (t, int((mask != img).sum()))
                assert ids == [0] + ecls and len(ids) == len(ecls) + 1, (t, ids, ecls)
                if t % 3 == 1 or t == len(fr) - 1:
                    ximg, xcls, _ = det.execute(rgb)
                    assert np.array_equal(ximg, img) and xcls == ecls, t
            else:
                assert ids == [] and not mask.any(), (t, tick, ids)
    finally:
        mf.attachDetector(None)
        mf.close()
    assert ran == len([t for t in range(1, N_FRAMES + 1) if _detect_runs(t, every_k)])


@pytest.mark.parametrize("on_device", [False, True], ids=["host", "device"])
def test_same_bits_as_mask_inputs(nets, frames, on_device):
    """a detector-driven context and a context fed its recorded masks as inputs agree on every frame and in the final surfel stores"""
    fr, _ = frames
    recs = _run_pair(nets(256), fr, None, 2, on_device)
    _check_handoff(recs)
    assert any(r["ran"] and len(r["ids"]) >= 2 for r in recs)


def test_oracle_parity_with_detector_masks(nets, frames):
    """the CPU oracle fed the masks the detector made agrees with the detector-driven context on every frame (test_gpu_multi.check_exact).
    Chosen so that objects are spawned from detector masks: scene seed 0 (table, 3 objects), S = 1024, default export (min_score 0.55),
    every_k = 1, modelSpawnOffset = 2, minRelSizeNew = 0.002 (KW)."""
    from tests.test_gpu_multi import MFS, check_exact
    det = nets(1024)
    fr, _ = frames
    orc = ol.OraclePipeline(ol.default_config(W, H, **KW))
    L = orc.L
    L.orc_mf_process_frame_ex.argtypes = [C.c_void_p] * 3 + [C.c_int64, C.c_void_p, C.c_void_p, C.c_int]
    mf = _ctx()
    mf.attachDetector(det, 1)
    log, most = [], 0
    try:
        for t, (rgb, depth, _) in enumerate(fr):
            mf.processFrame(rgb, depth, t * 33333)
            mask, ids = mf.frameMasks()
            most = max(most, len(ids) - 1)
            cls = np.array(ids, np.int32)
            L.orc_mf_process_frame_ex(orc.h, ol.ptr(rgb), ol.ptr(depth), t * 33333, ol.ptr(mask) if ids else None, ol.ptr(cls) if ids else None, len(ids))
            s = C.cast(orc.h, C.POINTER(MFS)).contents
            seg_c, proj_c = mf.segmentation()
            seg_o = ol.arr(s.mask, (H, W), np.uint8); proj_o = ol.arr(s.projectedIDs, (H, W), np.uint8)
            models_c = mf.getModels()
            rec = {"t": t, "n_o": int(s.nmodels), "n_c": len(models_c), "n_masks": len(ids),
                   "seg_diff": int((seg_c != seg_o).sum()), "proj_diff": int((proj_c != proj_o).sum()),
                   "ids_o": [int(orc.model(i).id) for i in range(s.nmodels)], "ids_c": [m.getID() for m in models_c],
                   "cls_o": [int(orc.model(i).classID) for i in range(s.nmodels)], "cls_c": [m.getClassID() for m in models_c],
                   "cnt_o": [int(orc.count(i)) for i in range(s.nmodels)], "cnt_c": [m.lastCount() for m in models_c]}
            if rec["n_o"] == rec["n_c"]:
                rec["dpose"] = [float(np.abs(orc.pose(i) - models_c[i].getPose()).max()) for i in range(rec["n_o"])]
            log.append(rec)
        n_final = int(C.cast(orc.h, C.POINTER(MFS)).contents.nmodels)
        log[-1]["traj"] = {"oracle": [np.array([orc.model(i).log[k] for k in range(orc.model(i).nlog * 8)]).reshape(-1, 8) for i in range(n_final)],
                           "cuda": [m.poseLog() for m in mf.getModels()]}
    finally:
        mf.attachDetector(None)
        mf.close()
    assert most >= 2, [r["n_masks"] for r in log]           # non-degenerate: some frame carries two or more detections
    check_exact(log, 2)                                      # >= 1 object model spawned from detector masks, every frame exact


def test_caller_mask_takes_precedence(nets, frames):
    """with a detector attached, frames given a mask use it and its classes and leave the detector alone; the results equal the context fed
    the same masks without a detector"""
    fr, cls = frames
    explicit = {4: True, 5: True, 9: True}
    recs = _run_pair(nets(256), fr, cls, 1, False, explicit)
    _check_handoff(recs)
    for r in recs:
        if r["given"]:
            assert np.array_equal(r["mask"], fr[r["t"]][2]) and r["ids"] == cls.tolist(), r["t"]
            assert np.array_equal(r["img"], r["before"][0]) and r["ecls"] == r["before"][1], r["t"]


def test_refusals(nets):
    import maskfusion_b200 as mfb
    import torch
    det = nets(256)
    bst = torch.cuda.Stream()
    bb = mfb.Backbone(256, seed=3, stream=bst.cuda_stream)
    st = _ctx(enableMultipleModels=0)
    L = st.L
    with pytest.raises(mfb.MFError, match="static"):
        st.attachDetector(det)
    with pytest.raises(mfb.MFError, match="static"):
        st.attachBackbone(bb, 5)
    st.attachBackbone(None)
    # a -static context never shards, not even as a one-rank communicator
    uid = (C.c_uint8 * 128)()
    assert L.mf_shard_unique_id(uid) == 0
    assert L.mf_shard_comm_init(st.h, uid, 0, 1) != 0 and "static" in L.mf_last_error().decode()
    st.close()
    mf = _ctx()
    L.mf_shard_configure.argtypes = [C.c_void_p, C.c_int, C.c_int]
    assert L.mf_shard_configure(mf.h, 0, 2) == 0
    with pytest.raises(mfb.MFError, match="sharded"):
        mf.attachDetector(det)
    mf.close()
    mf = _ctx()
    mf.attachBackbone(bb, 5)
    with pytest.raises(mfb.MFError, match="backbone is attached"):
        mf.attachDetector(det)
    mf.attachBackbone(None)
    mf.attachDetector(det)
    with pytest.raises(mfb.MFError, match="detector is attached"):
        mf.attachBackbone(bb, 5)
    assert L.mf_shard_configure(mf.h, 0, 2) != 0 and "detector" in L.mf_last_error().decode()
    assert L.mf_shard_comm_init(mf.h, uid, 0, 2) != 0 and "detector" in L.mf_last_error().decode()
    mf.attachDetector(None)
    mf.close()
    bb.close()


def test_export_error_surfaces_on_the_next_call(nets, frames):
    """special_assignments = [c] with c >= 1 an exported class: special_assignments[c] is out of range (IndexError upstream).  The frame
    runs without masks and the next call fails with the message"""
    import maskfusion_b200 as mfb
    det = nets(256)
    fr, _ = frames
    _, ecls, _ = det.execute(fr[1][0])
    assert ecls, "the detector exports nothing on frame 1"
    c = ecls[0]
    assert c >= 1
    det.set_export(special_assignments=[c])
    mf = _ctx()
    mf.attachDetector(det, 1)
    try:
        mf.processFrame(*fr[0][:2], 0)
        mf.processFrame(*fr[1][:2], 33333)                   # detects, the export rule fails on the device: the call itself succeeds
        with pytest.raises(mfb.MFError, match="special_assignments"):
            mf.sync()
        # the error is reported once; the failed frame carried no masks and the context goes on
        mask, ids = mf.frameMasks()
        assert ids == [] and not mask.any()
        det.set_export()
        mf.processFrame(*fr[2][:2], 2 * 33333)
        mask, ids = mf.frameMasks()
        assert ids and ids[0] == 0
    finally:
        mf.attachDetector(None)
        mf.close()
        det.set_export()


def test_detach_destroy_and_determinism(nets, frames):
    """detaching mid-run returns to mask-free frames; destroying a context with a detector attached is clean; two runs give the same bits"""
    det = nets(256)
    fr, _ = frames
    runs = []
    for rep in range(2):
        mf = _ctx()
        mf.attachDetector(det, 1)
        for t in range(6):
            mf.processFrame(*fr[t][:2], t * 33333)
        mf.sync()
        runs.append((_state(mf), mf.frameMasks(), _stores(mf)))
        if rep == 0:
            mf.attachDetector(None)
            for t in range(6, 9):
                mf.processFrame(*fr[t][:2], t * 33333)
                mask, ids = mf.frameMasks()
                assert ids == [] and not mask.any(), t
        mf.close()                                          # rep 1: destroyed with the detector still attached
    (a, ma, sa), (b, mb, sb) = runs
    _same_state(a, b, "rerun")
    assert np.array_equal(ma[0], mb[0]) and ma[1] == mb[1]
    assert all(np.array_equal(x, y) for x, y in zip(sa, sb))
    # the detector is still usable after the context that held it is gone
    img, ecls, _ = det.execute(fr[3][0])
    assert img.shape == (H, W)
