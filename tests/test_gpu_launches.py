"""The launches of a context: kernelLaunches() (mf_kernel_launches) counts every kernel the context enqueues, once, and its stage timer
(setProfiling / stageTimes) records the context's own launches whatever other contexts the process holds.

The count is checked against torch.profiler's CUDA trace.  The inputs are numpy arrays and no network is attached, so while the trace
runs nothing but the context launches a kernel, and every `kernel` record of the trace is one of its launches."""
from __future__ import annotations

import json

import numpy as np
import pytest

from tests.test_gpu_detect_frame import KW

pytestmark = pytest.mark.gpu
W, H = 640, 480
SW, SH = 320, 240                          # -static and stage-wise runs
STATIC_KW = dict(capacityGlobal=1000000, enableMultipleModels=0)
MULTI_KW = dict(KW, segMorphEdgeIterations=1, segMorphMaskIterations=1)


@pytest.fixture(scope="module")
def static_frames():
    from maskfusion_b200.synth import SynthScene
    sc = SynthScene(SW, SH, seed=1)
    return [tuple(np.ascontiguousarray(x) for x in sc.render(t)[:2]) for t in range(4)]


@pytest.fixture(scope="module")
def multi_frames():
    """the BASELINE configs[2] scene (table layout, three objects, seed 0), as tests/test_gpu_detect_frame.py"""
    from maskfusion_b200.synth import SynthScene
    sc = SynthScene(W, H, n_objects=3, seed=0, layout="table")
    out = []
    for t in range(10):
        rgb, depth, mask, *_ = sc.render(t)
        out.append((np.ascontiguousarray(rgb), np.ascontiguousarray(depth), np.ascontiguousarray(mask)))
    return out, np.array([0] + [o.class_id for o in sc.objects], np.int32)


def _static_ctx():
    import maskfusion_b200 as mfb
    return mfb.MaskFusion(mfb.default_config(SW, SH, **STATIC_KW))


def _kernels_traced(tmp_path, run):
    """run() -> a synchronised context it created; returns (its kernelLaunches(), the kernel records of the trace around run())"""
    import torch
    from torch.profiler import ProfilerActivity, profile
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        mf = run()
    try:
        counted = mf.kernelLaunches()
    finally:
        mf.close()
    path = tmp_path / "trace.json"
    prof.export_chrome_trace(str(path))
    events = json.loads(path.read_text())["traceEvents"]
    return counted, sum(1 for e in events if e.get("cat") == "kernel")


def test_static_frames(tmp_path, static_frames):
    def run():
        mf = _static_ctx()
        for t, (rgb, depth) in enumerate(static_frames):          # the first frame initialises the model, the others track it
            mf.processFrame(rgb, depth, t * 33333)
        mf.sync()
        return mf
    counted, traced = _kernels_traced(tmp_path, run)
    assert counted == traced


def test_multi_model_frames_that_spawn(tmp_path, multi_frames):
    import maskfusion_b200 as mfb
    fr, cls = multi_frames

    def run():
        mf = mfb.MaskFusion(mfb.default_config(W, H, **MULTI_KW))
        for t, (rgb, depth, mask) in enumerate(fr):
            mf.processFrame(rgb, depth, t * 33333, mask=mask, classIDs=cls)
        mf.sync()
        assert len(mf.getModels()) > 1                              # a model was spawned inside the run
        return mf
    counted, traced = _kernels_traced(tmp_path, run)
    assert counted == traced


def test_stage_calls_and_readbacks(tmp_path, static_frames):
    (rgb0, d0), (rgb1, d1) = static_frames[:2]

    def run():
        mf = _static_ctx()
        g = mf.getBackgroundModel()
        mf.setFrame(rgb0, d0)
        g.initialise(1)
        g.combinedPredict(1, 1)
        mf.setFrame(rgb1, d1)
        g.performTracking()
        g.predictIndices(2)
        g.fuse(2, 4.0)
        g.clean(2)
        g.combinedPredict(2, 2)
        g.overridePose(np.eye(4, dtype=np.float32))
        g.uploadMap(g.downloadMap())
        g.indexMap(); g.prediction(); g.fillIn(); g.association(); g.modelMaps(1); g.trackStats()
        mf.filteredDepth(); mf.frameMaps(1); mf.edgeMap()
        img = (rgb1[..., 0] > 128).astype(np.uint8) * 255
        mf.morphClose(img, 2, 1, ellipse=True)
        mf.morphClose(img, 1, 1, ellipse=False)
        mf.sync()
        return mf
    counted, traced = _kernels_traced(tmp_path, run)
    assert counted == traced


def test_stage_timer_belongs_to_its_context(static_frames):
    """a context created after profiling was turned on elsewhere does not take over the other context's marks"""
    rgb, depth = static_frames[0]
    a = _static_ctx()
    a.setProfiling(True)
    a.setFrame(rgb, depth)
    b = _static_ctx()
    try:
        a.getBackgroundModel().fuse(1, 4.0)
        a.sync()
        assert a.stageTimes()["k_associate"][0] == 1
    finally:
        b.close(); a.close()


def test_stage_timer_outlives_another_context(static_frames):
    """destroying another context between two stage-wise calls leaves both in this context's table"""
    rgb, depth = static_frames[0]
    a = _static_ctx()
    try:
        a.setProfiling(True)
        a.setFrame(rgb, depth)
        b = _static_ctx()
        g = a.getBackgroundModel()
        g.fuse(1, 4.0)
        b.close()
        g.clean(1)
        a.sync()
        st = a.stageTimes()
        assert st["k_associate"][0] == 1 and st["k_clean_p1"][0] == 1
    finally:
        a.close()
