"""The Mask R-CNN detector in the object-sharded mode (mf_shard_attach_detector / ShardedMaskFusion.attachDetector): the detector runs on
one rank and its frame mask + header reach every rank, so two shards compute what one process with MaskFusion.attachDetector computes,
bit for bit.

Two ranks, launched by torch.distributed.run on this file (the worker is at the bottom):
  - gloo, host-staged phases (mf_shard_frame_masks + dist.broadcast): always; both ranks may share cuda:0;
  - NCCL, the exchange inside the library (a fourth collective on detector frames): with two or more GPUs.
Checked: shards == one process on every frame (ids, classes, poses as bits, segmentation, projected ids, counts from the owner, frameMasks)
and in the final stores, for detector rank 1 and 0 with every_k 1 and 2; the ranks agree with each other; a caller's mask on rank 0 takes
precedence; an export error on the detector rank fails the next call on every rank and the run goes on; detaching; the collective count
(NCCL); the refusals of mf_shard_attach_detector."""
from __future__ import annotations

import ctypes as C
import os
import subprocess
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

from tests.test_cpu_sharding import free_port  # noqa: E402
from tests.test_gpu_detect_frame import KW, N_FRAMES, W, H  # noqa: E402

pytestmark = pytest.mark.gpu
P = W * H
# (name, detector rank, every_k, S, frames given the scene's mask + classes on rank 0)
SCENARIOS = [("r1k1", 1, 1, 256, ()), ("r1k2", 1, 2, 256, ()), ("r0k1", 0, 1, 256, ()), ("r0k2", 0, 2, 256, ()),
             ("given", 1, 1, 256, (4, 5, 9)), ("r1k1s1024", 1, 1, 1024, ())]


def scene_frames():
    from maskfusion_b200.synth import SynthScene
    sc = SynthScene(W, H, n_objects=3, seed=0, layout="table")
    out = []
    for t in range(N_FRAMES):
        rgb, depth, mask, *_ = sc.render(t)
        out.append((np.ascontiguousarray(rgb), np.ascontiguousarray(depth), np.ascontiguousarray(mask)))
    return out, np.array([0] + [o.class_id for o in sc.objects], np.int32)


def make_nets(S):
    """the seeded networks of tests/test_gpu_detect_frame.py (backbone 7, RPN 11, heads 13, export defaults) on a stream of their own"""
    import torch
    import maskfusion_b200 as mfb
    st = torch.cuda.Stream()
    bb = mfb.Backbone(S, seed=7, stream=st.cuda_stream)
    rpn = mfb.RegionProposals(bb, seed=11)
    det = mfb.Detector(rpn, seed=13)
    det.set_export()
    return st, bb, rpn, det


def close_nets(nets):
    for st, bb, rpn, det in nets.values():
        det.close(); rpn.close(); bb.close()


def record(out, key, mf, owner, rank):
    """what a frame decided, from one context (owner(i) == rank: the store is here; single process: owner = None)"""
    mf.sync()
    ms = mf.getModels()
    seg, proj = mf.segmentation()
    mask, ids = mf.frameMasks()
    own = [owner(i) if owner else 0 for i in range(len(ms))]
    out[f"{key}_ids"] = np.array([m.getID() for m in ms]); out[f"{key}_cls"] = np.array([m.getClassID() for m in ms])
    out[f"{key}_own"] = np.array(own)
    out[f"{key}_pose"] = np.stack([np.asarray(m.getPose(), np.float32).view(np.uint32) for m in ms])
    out[f"{key}_cnt"] = np.array([m.lastCount() if own[i] == rank else -1 for i, m in enumerate(ms)])
    out[f"{key}_seg"] = seg; out[f"{key}_proj"] = proj; out[f"{key}_mask"] = mask; out[f"{key}_mids"] = np.array(ids, np.int64)


def stores(out, name, mf, owner, rank):
    for i, m in enumerate(mf.getModels()):
        if (owner(i) if owner else 0) == rank:
            out[f"{name}_map{i}"] = np.ascontiguousarray(m.downloadMap()).view(np.uint32)


# ------------------------------------------------------------------------------------------------------------------------------------
# one process with attachDetector: the reference the shards must reproduce
# ------------------------------------------------------------------------------------------------------------------------------------
def single_run(det, fr, cls, every_k, given):
    import maskfusion_b200 as mfb
    mf = mfb.MaskFusion(mfb.default_config(W, H, **KW))
    mf.attachDetector(det, every_k)
    out = {}
    try:
        for t, (rgb, depth, smask) in enumerate(fr):
            if t in given:
                mf.processFrame(rgb, depth, t * 33333, mask=smask, classIDs=cls)
            else:
                mf.processFrame(rgb, depth, t * 33333)
            record(out, f"f{t}", mf, None, 0)
        stores(out, "end", mf, None, 0)
    finally:
        mf.attachDetector(None)
        mf.close()
    return out


def launch(backend, out_dir, timeout=1200):
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node=2", "--master-addr", "127.0.0.1",
           "--master-port", str(free_port()), os.path.abspath(__file__), backend, str(out_dir)]
    r = subprocess.run(cmd, capture_output=True, text=True, timeout=timeout, cwd=ROOT)
    assert r.returncode == 0, r.stdout[-3000:] + r.stderr[-3000:]
    return [dict(np.load(os.path.join(out_dir, f"rank{k}.npz"))) for k in range(2)]


@pytest.fixture(scope="module")
def reference():
    """single-process runs keyed by (S, every_k, given frames)"""
    fr, cls = scene_frames()
    nets = {S: make_nets(S) for S in sorted({s[3] for s in SCENARIOS})}
    try:
        refs = {}
        for _, _, k, S, given in SCENARIOS:
            if (S, k, given) not in refs:
                refs[(S, k, given)] = single_run(nets[S][3], fr, cls, k, given)
    finally:
        close_nets(nets)
    return refs


@pytest.fixture(scope="module", params=["gloo", "nccl"])
def shards(request, tmp_path_factory):
    import torch
    if request.param == "nccl" and torch.cuda.device_count() < 2:
        pytest.skip("the in-library NCCL exchange needs one GPU per rank")
    return request.param, launch(request.param, tmp_path_factory.mktemp(f"shard_detect_{request.param}"))


REPLICATED = ("ids", "cls", "own", "pose", "seg", "proj", "mask", "mids")


def test_shards_equal_one_process(shards, reference):
    """every scenario, every frame: both ranks equal the single process; counts from the owner; the stores on their owners"""
    _, ranks = shards
    spawned = []
    for name, _, k, S, given in SCENARIOS:
        ref = reference[(S, k, given)]
        for t in range(N_FRAMES):
            for key in ("ids", "cls", "pose", "seg", "proj", "mask", "mids"):
                for r in range(2):
                    a, b = ranks[r][f"{name}_f{t}_{key}"], ref[f"f{t}_{key}"]
                    assert a.shape == b.shape and np.array_equal(a, b), (name, t, key, r)
            cnt = np.where(ranks[0][f"{name}_f{t}_cnt"] >= 0, ranks[0][f"{name}_f{t}_cnt"], ranks[1][f"{name}_f{t}_cnt"])
            assert np.array_equal(cnt, ref[f"f{t}_cnt"]), (name, t, cnt, ref[f"f{t}_cnt"])
        owners = ranks[0][f"{name}_f{N_FRAMES - 1}_own"]
        for i in range(len(owners)):
            a, b = ranks[int(owners[i])][f"{name}_map{i}"], ref[f"end_map{i}"]
            assert a.shape == b.shape and np.array_equal(a, b), (name, i)
        if not given:
            spawned.append(max(len(ref[f"f{t}_ids"]) for t in range(N_FRAMES)) - 1)
    assert max(spawned) >= 1, ("no object model was spawned from detector masks", spawned)
    # the detector really ran: some frame carries two or more detections
    assert any(len(reference[(256, 1, ())][f"f{t}_mids"]) >= 2 for t in range(N_FRAMES))


def test_ranks_agree(shards):
    _, ranks = shards
    for name, *_ in SCENARIOS:
        for t in range(N_FRAMES):
            for key in REPLICATED:
                assert np.array_equal(ranks[0][f"{name}_f{t}_{key}"], ranks[1][f"{name}_f{t}_{key}"]), (name, t, key)


def test_caller_mask_takes_precedence(shards):
    """frames given the scene's mask + classes on rank 0 carry exactly those on both ranks, also when rank 1 detects"""
    _, ranks = shards
    fr, cls = scene_frames()
    given = dict((s[0], s[4]) for s in SCENARIOS)["given"]
    for t in given:
        for r in range(2):
            assert np.array_equal(ranks[r][f"given_f{t}_mask"], fr[t][2]), (t, r)
            assert ranks[r][f"given_f{t}_mids"].tolist() == cls.tolist(), (t, r)


def test_export_error_and_detach(shards):
    """special_assignments out of range on the detector rank: the next call fails with the message on EVERY rank, the failed frame carries
    no masks, the run goes on; after detaching on every rank, frames carry no masks"""
    _, ranks = shards
    for r in range(2):
        z = ranks[r]
        assert "special_assignments" in str(z["err_msg"]), (r, str(z["err_msg"]))
        assert z["err_after_ids"].tolist() == [] and not z["err_after_mask_any"], r
        assert z["err_next_ids"].tolist()[:1] == [0] and len(z["err_next_ids"]) >= 1, r
        assert all(not bool(v) for v in z["detached_any"]), r


def test_collective_count(shards):
    """NCCL: 3 collectives per tracking frame, a fourth on detector frames; it moves exactly width*height + sizeof(FrameHdr) bytes"""
    backend, ranks = shards
    if backend != "nccl":
        pytest.skip("calls are counted by the in-library NCCL exchange")
    z = ranks[0]
    for name, _, k, *_ in SCENARIOS:
        calls, nbytes = z[f"{name}_calls"], z[f"{name}_bytes"]
        assert calls[0] == 1, (name, calls)                                    # tick 1: the packet only
        for t in range(1, N_FRAMES):
            assert calls[t] == 3 + int((t + 1) % k == 0), (name, t, calls)
        hdr = int(nbytes[0]) - 8 * P                                            # the packet is rgb | depth | mask | FrameHdr
        if k == 2:
            assert int(nbytes[3]) - int(nbytes[2]) == P + hdr, (name, nbytes)   # tick 4 exchanges, tick 3 does not


def test_refusals():
    """mf_shard_attach_detector: -static, world == 1, detector_rank out of range, a detector on the wrong rank / none on the detector rank,
    a backbone attached; the single-process refusals still hold with a shard detector attached"""
    import torch
    import maskfusion_b200 as mfb
    nets = {256: make_nets(256)}
    det = nets[256][3]
    L = mfb.load_library()

    def refused(mf, d, k, r, text):
        assert L.mf_shard_attach_detector(mf.h, C.c_void_p(d.h) if d else None, k, r) != 0
        assert text in L.mf_last_error().decode(), L.mf_last_error().decode()

    ctxs = []

    def ctx(rank=None, **over):
        kw = dict(KW); kw.update(over)
        mf = mfb.MaskFusion(mfb.default_config(W, H, **kw)); ctxs.append(mf)
        if rank is not None:
            assert L.mf_shard_configure(mf.h, rank, 2) == 0
        return mf

    bst = torch.cuda.Stream()
    bb = mfb.Backbone(256, seed=3, stream=bst.cuda_stream)
    try:
        refused(ctx(enableMultipleModels=0), det, 1, 0, "static")
        refused(ctx(), det, 1, 0, "mf_attach_detector")                     # world == 1
        a = ctx(0)
        refused(a, det, 1, 2, "outside [0, 2)")
        refused(a, det, 1, -1, "outside [0, 2)")
        refused(a, det, 1, 1, "not the detector rank")
        refused(ctx(1), None, 1, 1, "no detector given")
        a.attachBackbone(bb, 5)
        refused(a, det, 1, 0, "backbone")
        a.attachBackbone(None)
        assert L.mf_shard_attach_detector(a.h, C.c_void_p(det.h), 2, 0) == 0
        b = ctx(1)
        assert L.mf_shard_attach_detector(b.h, None, 2, 0) == 0                 # a rank without the detector
        for m in (a, b):
            with pytest.raises(mfb.MFError, match="sharded"):
                m.attachDetector(det)
            with pytest.raises(mfb.MFError, match="detector is attached"):
                m.attachBackbone(bb, 5)
            assert L.mf_shard_configure(m.h, 0, 2) != 0 and "detector" in L.mf_last_error().decode()
            assert L.mf_shard_attach_detector(m.h, None, 0, -1) == 0           # detach
            m.attachBackbone(bb, 5); m.attachBackbone(None)
    finally:
        for mf in ctxs:
            mf.close()
        bb.close()
        close_nets(nets)


# ------------------------------------------------------------------------------------------------------------------------------------
# worker: one rank (python -m torch.distributed.run --nproc-per-node 2 tests/test_gpu_shard_detect.py <gloo|nccl> <out_dir>)
# ------------------------------------------------------------------------------------------------------------------------------------
def worker(backend, out_dir):
    import torch
    import torch.distributed as dist
    import maskfusion_b200 as mfb
    from maskfusion_b200.sharding import ShardedMaskFusion
    rank, world = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"])
    dev = int(os.environ.get("LOCAL_RANK", 0)) if torch.cuda.device_count() >= world else 0
    torch.cuda.set_device(dev)
    if backend == "nccl":
        dist.init_process_group("nccl", device_id=torch.device("cuda", dev))
    else:
        dist.init_process_group("gloo")
    fr, cls = scene_frames() if rank == 0 else (None, None)
    nets = {S: make_nets(S) for S in sorted({s[3] for s in SCENARIOS})}
    out = {}

    def frame(smf, t, given=False):
        if rank == 0:
            rgb, depth, smask = fr[t]
            smf.processFrame(rgb, depth, t * 33333, mask=smask if given else None, classIDs=cls if given else None)
        else:
            smf.processFrame()

    def shard():
        return ShardedMaskFusion(mfb.default_config(W, H, **KW), device=dev)

    for name, det_rank, k, S, given in SCENARIOS:
        smf = shard()
        smf.attachDetector(nets[S][3], k, det_rank)
        calls, nbytes = [], []
        for t in range(N_FRAMES):
            s0 = smf.stats()
            frame(smf, t, t in given)
            smf.mf.sync()
            s1 = smf.stats()
            calls.append((s1["calls"] or 0) - (s0["calls"] or 0)); nbytes.append(s1["bytes"] - s0["bytes"])
            record(out, f"{name}_f{t}", smf.mf, smf.owner, rank)
        stores(out, name, smf.mf, smf.owner, rank)
        out[f"{name}_calls"] = np.array(calls); out[f"{name}_bytes"] = np.array(nbytes)
        smf.detachDetector()
        smf.close()

    # export error on the detector rank (1), then detaching
    det = nets[256][3]
    smf = shard()
    smf.attachDetector(det, 1, 1)
    frame(smf, 0)
    if rank == 1:
        from maskfusion_b200.synth import SynthScene
        _, ecls, _ = det.execute(np.ascontiguousarray(SynthScene(W, H, n_objects=3, seed=0, layout="table").render(1)[0]))
        assert ecls and ecls[0] >= 1, ecls
        det.set_export(special_assignments=[ecls[0]])
    frame(smf, 1)                                            # detects; the export rule fails on the device: the call itself succeeds
    msg = ""
    try:
        smf.mf.sync()
    except mfb.MFError as e:
        msg = str(e)
    out["err_msg"] = np.array(msg)
    mask, ids = smf.frameMasks()
    out["err_after_ids"] = np.array(ids, np.int64); out["err_after_mask_any"] = np.array(bool(mask.any()))
    if rank == 1:
        det.set_export()
    frame(smf, 2)
    out["err_next_ids"] = np.array(smf.frameMasks()[1], np.int64)
    smf.detachDetector()
    detached = []
    for t in (3, 4):
        frame(smf, t)
        mask, ids = smf.frameMasks()
        detached.append(bool(ids) or bool(mask.any()))
    out["detached_any"] = np.array(detached)
    smf.close()
    close_nets(nets)
    np.savez(os.path.join(out_dir, f"rank{rank}.npz"), **out)
    dist.destroy_process_group()


if __name__ == "__main__":
    os.makedirs(sys.argv[2], exist_ok=True)
    worker(sys.argv[1], sys.argv[2])
