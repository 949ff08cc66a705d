"""Contexts and Mask R-CNN handles driven from several threads of one process compute what each computes alone.  What the library keeps
per device (SM count, occupancies, kernel attributes), per context (the tracker's flag epoch) and process-wide under a lock (the GEMM's
tensor maps) must not leak from one of them into another:

  - two -static contexts on differently noisy frames and one seeded backbone forward run one after another on the main thread, then once
    together from three threads released by one barrier: every pose log, pose, surfel map and P2..P6 level is the same, bit for bit.  The
    tracker's cooperative grid then runs next to the other context's frames and the backbone's GEMMs;
  - with two GPUs, in a process of its own: a backbone on device 0, then a context on device 1, then the backbone again on device 0 give
    the bits of the same work on device 0 alone."""
from __future__ import annotations

import hashlib
import json
import os
import subprocess
import sys
import threading

import numpy as np
import pytest

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SW, SH, FRAMES, S = 320, 240, 8, 256
STATIC_KW = dict(capacityGlobal=1000000, enableMultipleModels=0)
SEEDS = (1, 2)


def _sha(a: np.ndarray) -> str:
    return hashlib.sha256(np.ascontiguousarray(a).tobytes()).hexdigest()


def frames(seed):
    """the seed sets the depth noise: the room is the same for every seed"""
    from maskfusion_b200.synth import SynthScene
    sc = SynthScene(SW, SH, seed=seed, noise=True)
    return [tuple(np.ascontiguousarray(x) for x in sc.render(t)[:2]) for t in range(FRAMES)]


def backbone_input(device=0):
    import torch
    g = torch.Generator(device="cpu").manual_seed(5)
    x = (torch.rand(S, S, 3, generator=g) * 200 - 100).to(torch.bfloat16).cuda(device)
    torch.cuda.synchronize(device)
    return x


def context_job(scene, device=0):
    """digests of the pose log, pose and surfel map of a -static context on `device`, and the number of surfels"""
    import maskfusion_b200 as mfb
    mf = mfb.MaskFusion(mfb.default_config(SW, SH, **STATIC_KW), device=device)
    try:
        for t, (rgb, depth) in enumerate(scene):
            mf.processFrame(rgb, depth, t * 33333)
        mf.sync()
        g = mf.getBackgroundModel()
        surfels = g.downloadMap()
        return [_sha(g.poseLog()), _sha(np.float32(g.getPose())), _sha(np.float32(surfels)), int(surfels.shape[0])]
    finally:
        mf.close()


def backbone_job(x):
    """digests of P2..P6 of a seeded backbone's forward on x, on a stream of its own on x's device (the thread's current device)"""
    import torch
    import maskfusion_b200 as mfb
    bb = mfb.Backbone(S, seed=7, stream=torch.cuda.Stream(x.device).cuda_stream)
    try:
        bb.forward(x.data_ptr())
        return [_sha(bb.download(level)) for level in range(4, 9)]
    finally:
        bb.close()


def test_two_contexts_and_a_backbone_on_three_threads():
    scenes = [frames(seed) for seed in SEEDS]
    x = backbone_input()
    jobs = [lambda s=s: context_job(s) for s in scenes] + [lambda: backbone_job(x)]
    alone = [job() for job in jobs]
    assert all(r[3] > 0 for r in alone[:2]) and alone[0] != alone[1]

    together, barrier = [None] * len(jobs), threading.Barrier(len(jobs), timeout=120)

    def run(i):
        try:
            barrier.wait()
            together[i] = jobs[i]()
        except BaseException as e:          # noqa: BLE001 -- reported by the main thread
            together[i] = e

    threads = [threading.Thread(target=run, args=(i,)) for i in range(len(jobs))]
    for t in threads:
        t.start()
    for t in threads:
        t.join()
    names = [["pose log", "pose", "surfel map", "surfels"]] * 2 + [["P%d" % p for p in range(2, 7)]]
    for i, (got, want) in enumerate(zip(together, alone)):
        assert not isinstance(got, BaseException), (i, repr(got))
        assert got == want, (i, [n for n, a, b in zip(names[i], got, want) if a != b])


_TWO_DEVICES = r"""
import json
import torch
from tests.test_gpu_shared_state import SEEDS, backbone_input, backbone_job, context_job, frames
torch.cuda.set_device(0)
x = backbone_input(0)
first = backbone_job(x)
ctx = context_job(frames(SEEDS[0]), device=1)
torch.cuda.set_device(0)
again = backbone_job(x)
print(json.dumps([ctx, first, again]))
"""


def test_a_context_on_a_second_device():
    import torch
    if torch.cuda.device_count() < 2:
        pytest.skip("needs two CUDA devices")
    ctx0, bb0 = context_job(frames(SEEDS[0])), backbone_job(backbone_input())
    r = subprocess.run([sys.executable, "-c", _TWO_DEVICES], capture_output=True, text=True, cwd=ROOT, timeout=600)
    assert r.returncode == 0, r.stderr
    ctx1, first, again = json.loads(r.stdout.strip().splitlines()[-1])
    assert ctx1 == ctx0
    assert first == bb0 and again == bb0
