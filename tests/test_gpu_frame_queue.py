"""The frame queue (mf_set_frame_queue / MaskFusion.setFrameQueue, the reference's -frameQ, MaskFusion.cpp:200-209).

A queued run of N calls processes the first N - length + 1 frames, frame m at tick m + 1, exactly as an unqueued run of those frames:
  - -static, host and device inputs: pose logs (bits), surfel stores, index map and prediction;
  - the call-bound arguments (inPose, bootstrap, weightMultiplier) apply to the frame the call processes;
  - multi-model with the scene's masks and classes: every processed frame, with objects spawned inside the queued run;
  - with the detector attached (detection at push time): masks, poses, segmentation and stores of every processed frame; a caller's mask
    still wins; an export error fails the call after the frame is processed; detaching and destroying with frames queued;
  - the refusals; length 0 and 1 are the unqueued path."""
from __future__ import annotations

import ctypes as C

import numpy as np
import pytest

from tests.test_gpu_detect_frame import KW, _same_state, _state, _stores

pytestmark = pytest.mark.gpu
W, H = 640, 480
SW, SH = 320, 240                          # -static runs
STATIC_KW = dict(capacityGlobal=1000000, enableMultipleModels=0)
N_DET = 36                                 # frames rendered for the multi-model legs: a queue of 30 still processes 7 of them


@pytest.fixture(scope="module")
def static_frames():
    from maskfusion_b200.synth import SynthScene
    sc = SynthScene(SW, SH, seed=1)
    return [tuple(np.ascontiguousarray(x) for x in sc.render(t)[:2]) for t in range(36)]


@pytest.fixture(scope="module")
def multi_frames():
    """the BASELINE configs[2] scene (table layout, three objects, seed 0), as tests/test_gpu_detect_frame.py"""
    from maskfusion_b200.synth import SynthScene
    sc = SynthScene(W, H, n_objects=3, seed=0, layout="table")
    out = []
    for t in range(N_DET):
        rgb, depth, mask, *_ = sc.render(t)
        out.append((np.ascontiguousarray(rgb), np.ascontiguousarray(depth), np.ascontiguousarray(mask)))
    return out, np.array([0] + [o.class_id for o in sc.objects], np.int32)


@pytest.fixture(scope="module")
def nets():
    """S -> Detector (the seeded weights of tests/test_gpu_detect_frame.py) on a stream of its own"""
    import torch
    import maskfusion_b200 as mfb
    made = {}

    def get(S):
        if S not in made:
            st = torch.cuda.Stream()
            bb = mfb.Backbone(S, seed=7, stream=st.cuda_stream)
            rpn = mfb.RegionProposals(bb, seed=11)
            made[S] = (st, bb, rpn, mfb.Detector(rpn, seed=13))
        det = made[S][3]
        det.set_export()
        return det

    yield get
    for st, bb, rpn, det in made.values():
        det.close(); rpn.close(); bb.close()


def _static_ctx(queue=None, stream=None):
    import maskfusion_b200 as mfb
    mf = mfb.MaskFusion(mfb.default_config(SW, SH, **STATIC_KW), stream=stream)
    if queue is not None:
        mf.setFrameQueue(queue)
    return mf


def _multi_ctx(queue=None, **over):
    import maskfusion_b200 as mfb
    kw = dict(KW); kw.update(over)
    mf = mfb.MaskFusion(mfb.default_config(W, H, **kw))
    if queue is not None:
        mf.setFrameQueue(queue)
    return mf


def _static_final(mf):
    """everything a -static run leaves: pose log and pose as bits, the store, index map and prediction of the global model"""
    g = mf.getBackgroundModel()
    mf.sync()
    return {"log": g.poseLog().view(np.uint64).copy(), "pose": np.asarray(g.getPose(), np.float32).view(np.uint32).copy(),
            "store": np.ascontiguousarray(g.downloadMap()).view(np.uint32).copy(),
            "index": [np.ascontiguousarray(a).view(np.uint32).copy() for a in g.indexMap()],
            "pred": [np.ascontiguousarray(a).view(np.uint8).copy() for a in g.prediction()], "tick": mf.getTick()}


def _same_static(a, b):
    assert a["tick"] == b["tick"]
    assert a["log"].shape == b["log"].shape and np.array_equal(a["log"], b["log"])
    assert np.array_equal(a["pose"], b["pose"])
    assert a["store"].shape == b["store"].shape and np.array_equal(a["store"], b["store"])
    assert all(np.array_equal(x, y) for x, y in zip(a["index"], b["index"]))
    assert all(np.array_equal(x, y) for x, y in zip(a["pred"], b["pred"]))


def _static_run(fr, queue, calls, on_device, args=None):
    """`calls` calls of a -static context (queue None: never set); args: {call: kwargs of processFrame}.  Device inputs are written into ONE
    pair of device buffers that every call reuses right after it returns (the copy into the queue slot happens at push time)."""
    import torch
    st = torch.cuda.Stream() if on_device else None
    mf = _static_ctx(queue, st.cuda_stream if st is not None else None)
    sizes = []
    try:
        if on_device:
            rgb_d = torch.empty((SH, SW, 3), dtype=torch.uint8, device="cuda")
            dep_d = torch.empty((SH, SW), dtype=torch.float32, device="cuda")
        for c in range(calls):
            rgb, depth = fr[c]
            kw = (args or {}).get(c, {})
            if on_device:
                assert not kw
                with torch.cuda.stream(st):                 # behind the previous call's copies (they are ordered on the context stream)
                    rgb_d.copy_(torch.from_numpy(rgb), non_blocking=False); dep_d.copy_(torch.from_numpy(depth), non_blocking=False)
                st.synchronize()
                mf.processFramePtr(rgb_d.data_ptr(), dep_d.data_ptr(), c * 33333, True)
            else:
                mf.processFrame(rgb, depth, c * 33333, **kw)
            sizes.append((mf.getTick(), mf.frameQueueSize()))
        return _static_final(mf), sizes
    finally:
        mf.close()


@pytest.mark.parametrize("on_device", [False, True], ids=["host", "device"])
@pytest.mark.parametrize("length", [2, 5, 30])
def test_static_shift_equivalence(static_frames, length, on_device):
    n = length + 5
    q, sizes = _static_run(static_frames, length, n, on_device)
    ref, _ = _static_run(static_frames, None, n - length + 1, on_device)
    _same_static(q, ref)
    # the filling calls: nothing processed, the queue counts up; then one frame per call and length - 1 frames stay queued
    assert sizes[:length - 1] == [(1, c + 1) for c in range(length - 1)], sizes
    assert sizes[length - 1:] == [(c + 2, length - 1) for c in range(n - length + 1)], sizes
    assert len(q["log"]) == n - length + 1


def test_call_bound_arguments(static_frames):
    """inPose / bootstrap / weightMultiplier of a call apply to the frame the call processes (as the reference's processFrame)"""
    length, n = 4, 16
    T = np.eye(4, dtype=np.float32); T[0, 3] = 0.01; T[2, 3] = -0.02
    B = np.eye(4, dtype=np.float32); B[1, 3] = 0.005
    call_args = {5: dict(inPose=T), 6: dict(weightMultiplier=0.5), 8: dict(inPose=B, bootstrap=True), 9: dict(weightMultiplier=3.0),
                 12: dict(inPose=T, weightMultiplier=2.0)}
    q, _ = _static_run(static_frames, length, n, False, call_args)
    shifted = {c - (length - 1): kw for c, kw in call_args.items()}
    ref, _ = _static_run(static_frames, None, n - length + 1, False, shifted)
    _same_static(q, ref)


@pytest.mark.parametrize("length", [0, 1])
def test_no_queue_is_the_unqueued_path(static_frames, multi_frames, length):
    a, _ = _static_run(static_frames, length, 8, False)
    b, _ = _static_run(static_frames, None, 8, False)
    _same_static(a, b)
    fr, cls = multi_frames
    A, B = _multi_ctx(length), _multi_ctx()
    try:
        for t in range(8):
            for mf in (A, B):
                mf.processFrame(fr[t][0], fr[t][1], t * 33333, mask=fr[t][2], classIDs=cls)
                assert mf.frameQueueSize() == 0
            A.sync(); B.sync()
            _same_state(_state(A), _state(B), t)
        sa, sb = _stores(A), _stores(B)
        assert len(sa) == len(sb) and all(np.array_equal(x, y) for x, y in zip(sa, sb))
    finally:
        A.close(); B.close()


def _lockstep(A, B, length, fr, n, feed, check=None):
    """call c of the queued context A pushes frame c; once it processes frame m = c - length + 1, the unqueued context B processes frame m
    and both are compared.  feed(mf, t, queued) issues the processFrame call of frame t."""
    for c in range(n):
        feed(A, c, True)
        m = c - length + 1
        if m < 0:
            assert A.getTick() == 1 and A.frameQueueSize() == c + 1
            continue
        feed(B, m, False)
        A.sync(); B.sync()
        assert A.getTick() == B.getTick() == m + 2 and A.frameQueueSize() == length - 1
        _same_state(_state(A), _state(B), m)
        assert np.array_equal(A.getBackgroundModel().poseLog().view(np.uint64), B.getBackgroundModel().poseLog().view(np.uint64)), m
        if check:
            check(m)
    sa, sb = _stores(A), _stores(B)
    assert len(sa) == len(sb) and all(np.array_equal(x, y) for x, y in zip(sa, sb))
    return len(sa)


@pytest.mark.parametrize("length", [3, 30])
def test_multi_model_with_masks(multi_frames, length):
    """the scene's masks with setFrameClasses before each call: the classes travel with the queued frame"""
    fr, cls = multi_frames
    n = min(len(fr), length + 12)
    A, B = _multi_ctx(length), _multi_ctx()

    def feed(mf, t, queued):
        mf.setFrameClasses(cls)
        mf.processFrame(fr[t][0], fr[t][1], t * 33333, mask=fr[t][2])
        mf.setFrameClasses([])                  # the next call sets its own: a stale list must not reach a queued frame

    try:
        models = _lockstep(A, B, length, fr, n, feed)
    finally:
        A.close(); B.close()
    assert models > 1                            # objects spawned inside the queued run


@pytest.mark.parametrize("length", [3, 30])
@pytest.mark.parametrize("every_k", [1, 2])
@pytest.mark.parametrize("S", [256, 1024])
def test_detector_attached(nets, multi_frames, S, every_k, length):
    """detection at push time equals the unqueued detector run, frame by frame; with length 3 some frames carry the caller's mask"""
    det = nets(S)
    fr, cls = multi_frames
    n = min(len(fr), length + 10)
    explicit = {4, 5, 9} if length == 3 else set()
    A, B = _multi_ctx(length), _multi_ctx()
    A.attachDetector(det, every_k); B.attachDetector(det, every_k)

    def feed(mf, t, queued):
        if t in explicit:
            mf.setFrameClasses(cls)
            mf.processFrame(fr[t][0], fr[t][1], t * 33333, mask=fr[t][2])
        else:
            mf.processFrame(fr[t][0], fr[t][1], t * 33333)

    ran = []

    def check(m):
        ma, ia = A.frameMasks(); mb, ib = B.frameMasks()
        assert ia == ib and np.array_equal(ma, mb), m
        if m in explicit:
            assert ia == cls.tolist() and np.array_equal(ma, fr[m][2]), m
        elif m + 1 > 1 and (m + 1) % every_k == 0:
            ran.append(len(ia))
        else:
            assert ia == [] and not ma.any(), m

    try:
        _lockstep(A, B, length, fr, n, feed, check)
    finally:
        A.attachDetector(None); B.attachDetector(None)
        A.close(); B.close()
    assert ran and any(k >= 2 for k in ran), ran


def test_export_error_after_the_frame_is_processed(nets, multi_frames):
    import maskfusion_b200 as mfb
    det = nets(256)
    fr, _ = multi_frames
    _, ecls, _ = det.execute(fr[1][0])
    assert ecls and ecls[0] >= 1
    mf = _multi_ctx(3)
    mf.attachDetector(det, 1)
    try:
        det.set_export(special_assignments=[ecls[0]])
        mf.processFrame(*fr[0][:2], 0)
        mf.processFrame(*fr[1][:2], 33333)          # frame 1 is detected at push time, with the failing rule
        det.set_export()
        mf.processFrame(*fr[2][:2], 2 * 33333)      # processes frame 0
        mf.sync()
        mf.processFrame(*fr[3][:2], 3 * 33333)      # processes frame 1: the call succeeds, the error surfaces on the next one
        with pytest.raises(mfb.MFError, match="special_assignments.*timestamp 33333"):
            mf.sync()
        mask, ids = mf.frameMasks()
        assert ids == [] and not mask.any()
        mf.processFrame(*fr[4][:2], 4 * 33333)      # processes frame 2, detected with the default rule
        mask, ids = mf.frameMasks()
        assert ids and ids[0] == 0
    finally:
        mf.attachDetector(None)
        mf.close()
        det.set_export()


def test_detach_and_destroy_with_frames_queued(nets, multi_frames):
    import torch
    det = nets(1024)
    fr, _ = multi_frames
    mf = _multi_ctx(8)
    mf.attachDetector(det, 1)
    for t in range(6):                                # frames 1..5 are being detected
        mf.processFrame(*fr[t][:2], t * 33333)
    assert mf.frameQueueSize() == 6 and mf.getTick() == 1
    mf.attachDetector(None)                           # waits for the hand-offs into the queued frames
    for t in range(6, 12):
        mf.processFrame(*fr[t][:2], t * 33333)
        mask, ids = mf.frameMasks()
        m = t - 7                                      # the processed frame
        if m >= 1:
            assert ids and ids[0] == 0, (t, m)        # detected before the detach
        else:
            assert ids == [] and not mask.any(), (t, m)
    mf.close()
    # destroyed with frames queued and detections in flight
    mf = _multi_ctx(30)
    mf.attachDetector(det, 1)
    for t in range(8):
        mf.processFrame(*fr[t][:2], t * 33333)
    mf.close()
    torch.cuda.synchronize()
    img, ecls, _ = det.execute(fr[3][0])              # the detector is usable and no work is left behind
    assert img.shape == (H, W)


def test_refusals(static_frames):
    import maskfusion_b200 as mfb
    fr = static_frames
    L = mfb.load_library()
    L.mf_shard_configure.argtypes = [C.c_void_p, C.c_int, C.c_int]
    L.mf_set_frame.argtypes = [C.c_void_p] * 4
    mf = _static_ctx()
    with pytest.raises(mfb.MFError, match=">= 0"):
        mf.setFrameQueue(-1)
    mf.setFrameQueue(4)                               # a refused call leaves the context usable
    for t in range(2):
        mf.processFrame(*fr[t], t * 33333)
    with pytest.raises(mfb.MFError, match="before the first frame"):
        mf.setFrameQueue(2)
    with pytest.raises(mfb.MFError, match="queued"):
        mf.setFrame(*fr[0])
    g = mf.getBackgroundModel()
    for call in (lambda: L.mf_model_predict_indices(mf.h, 0, 1), lambda: L.mf_model_fuse(mf.h, 0, 1, C.c_float(4.0), C.c_float(1.0)),
                 lambda: L.mf_model_clean(mf.h, 0, 1), lambda: L.mf_model_combined_predict(mf.h, 0, 1, 1),
                 lambda: L.mf_model_init_from_frame(mf.h, 0, 1), lambda: L.mf_model_perform_tracking(mf.h, 0, None)):
        assert call() != 0 and "queued" in L.mf_last_error().decode()
    for t in range(2, 6):
        mf.processFrame(*fr[t], t * 33333)
    assert mf.getTick() == 4 and mf.frameQueueSize() == 3 and g.lastCount() > 0
    mf.close()
    # sharded contexts, both ways round
    mm = _multi_ctx()
    assert L.mf_shard_configure(mm.h, 0, 2) == 0
    with pytest.raises(mfb.MFError, match="sharded"):
        mm.setFrameQueue(5)
    mm.close()
    mm = _multi_ctx(5)
    assert L.mf_shard_configure(mm.h, 0, 2) != 0 and "frame queue" in L.mf_last_error().decode()
    uid = (C.c_uint8 * 128)()
    assert L.mf_shard_unique_id(uid) == 0
    assert L.mf_shard_comm_init(mm.h, uid, 0, 2) != 0 and "frame queue" in L.mf_last_error().decode()
    mm.close()


def test_in_pose_call_reads_the_detected_masks(nets, multi_frames):
    """a queued frame is detected at push time; when the call that pops it passes an inPose the frame does not segment, and frameMasks()
    still returns the completed hand-off (it waits for the frame's detection)"""
    det = nets(256)
    fr, _ = multi_frames
    length = 3
    mf = _multi_ctx(length)
    mf.attachDetector(det, 1)
    try:
        for c in range(8):
            kw = dict(inPose=np.eye(4, dtype=np.float32)) if c == 6 else {}
            mf.processFrame(*fr[c][:2], c * 33333, **kw)
            m = c - length + 1
            if c == 6:
                mask, ids = mf.frameMasks()
                img, ecls, _ = det.execute(fr[m][0])
                assert ids == [0] + ecls and np.array_equal(mask, img), (m, ids, ecls)
        mf.sync()
    finally:
        mf.attachDetector(None)
        mf.close()
