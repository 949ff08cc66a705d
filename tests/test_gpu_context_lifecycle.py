"""Creating and destroying contexts: every stream, event and pinned buffer a context owns is released with it, and what it borrows is not.

  - a -static context on the caller's stream, closed, then a second one on the same stream: the same bits, and the caller's stream still
    runs work afterwards (the context never destroyed it);
  - a multi-model context with the stage timer on and a frame queue, long enough to spawn an object model, created and closed twice in one
    process: the same poses, model ids and stage table."""
from __future__ import annotations

import numpy as np
import pytest

from tests.test_gpu_detect_frame import KW

pytestmark = pytest.mark.gpu
W, H = 640, 480
SW, SH = 320, 240
STATIC_KW = dict(capacityGlobal=1000000, enableMultipleModels=0)


def _bits(a):
    return np.ascontiguousarray(a, np.float32).view(np.uint32).copy()


def _static_run(stream, frames):
    import maskfusion_b200 as mfb
    mf = mfb.MaskFusion(mfb.default_config(SW, SH, **STATIC_KW), stream=stream.cuda_stream)
    try:
        for t, (rgb, depth) in enumerate(frames):
            mf.processFrame(rgb, depth, t * 33333)
        mf.sync()
        g = mf.getBackgroundModel()
        return g.poseLog().copy(), _bits(g.getPose()), _bits(g.downloadMap())
    finally:
        mf.close()


def test_static_contexts_on_the_callers_stream():
    import torch
    from maskfusion_b200.synth import SynthScene
    sc = SynthScene(SW, SH, seed=1)
    frames = [tuple(np.ascontiguousarray(x) for x in sc.render(t)[:2]) for t in range(5)]
    st = torch.cuda.Stream()
    a = _static_run(st, frames)
    b = _static_run(st, frames)
    assert np.array_equal(a[0].view(np.uint64), b[0].view(np.uint64))
    assert np.array_equal(a[1], b[1]) and np.array_equal(a[2], b[2])
    assert a[2].shape[0] > 0
    with torch.cuda.stream(st):
        y = (torch.arange(1000, device="cuda", dtype=torch.int64) * 2).sum()
    st.synchronize()
    assert y.item() == 999000


def _multi_run(frames, cls):
    import maskfusion_b200 as mfb
    mf = mfb.MaskFusion(mfb.default_config(W, H, **KW))
    try:
        mf.setProfiling(True)
        mf.setFrameQueue(3)
        for t, (rgb, depth, mask) in enumerate(frames):
            mf.processFrame(rgb, depth, t * 33333, mask=mask, classIDs=cls)
        mf.sync()
        ms = mf.getModels()
        return ([m.getID() for m in ms], [_bits(m.getPose()) for m in ms], {k: v[0] for k, v in mf.stageTimes().items()})
    finally:
        mf.close()


def test_multi_model_contexts_twice():
    from maskfusion_b200.synth import SynthScene
    sc = SynthScene(W, H, n_objects=3, seed=0, layout="table")
    frames = []
    for t in range(12):
        rgb, depth, mask, *_ = sc.render(t)
        frames.append((np.ascontiguousarray(rgb), np.ascontiguousarray(depth), np.ascontiguousarray(mask)))
    cls = np.array([0] + [o.class_id for o in sc.objects], np.int32)
    ids_a, poses_a, stages_a = _multi_run(frames, cls)
    ids_b, poses_b, stages_b = _multi_run(frames, cls)
    assert len(ids_a) > 1, ids_a                              # an object model was spawned
    assert ids_a == ids_b
    assert all(np.array_equal(x, y) for x, y in zip(poses_a, poses_b))
    assert stages_a == stages_b and "k_associate" in stages_a
