#!/usr/bin/env python
"""The Mask R-CNN detector in the object-sharded mode (mf_shard_attach_detector) against masks as inputs and against one process.

    torchrun --nproc-per-node N scripts/bench_shard_detect.py      (N >= 2, one GPU per rank, NCCL)

bench.py's sharded configs[3] set-up: the table scene with 8 objects, MULTI_KW, 640x480, device-resident inputs on rank 0, frames
[0, --timed-from) as warm-up, then CUDA events around frames [--timed-from, --frames), the slowest rank's time.  Legs:
  shard_masks              the scene's masks + classes as inputs, no detector (bench.py's configs[3] path)
  shard_det1024_k1 / _k5   detector at S = 1024 on rank N-1, every_k 1 and 5, no masks given
  single_det1024_k1 / _k5  the same detector legs in one process on rank 0's GPU (the baseline)
Per leg: ms per frame, frames/s, the model count, and for the sharded legs the NCCL calls and bytes per frame.  Detector masks spawn other
models than the scene's masks, so the workloads of the masks and detector legs differ.  The legs run --repeats times in alternating
order; the spread over the repeats is printed.  One JSON object from rank 0, with the GPU name and power limit read in the same run."""
import argparse
import datetime
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import numpy as np

W, H = 640, 480
SHARD_LEGS = [("shard_masks", 0), ("shard_det1024_k1", 1), ("shard_det1024_k5", 5)]
SINGLE_LEGS = [("single_det1024_k1", 1), ("single_det1024_k5", 5)]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", type=int, default=60)
    ap.add_argument("--timed-from", type=int, default=20)
    ap.add_argument("--repeats", type=int, default=2)
    a = ap.parse_args()
    rank, world = int(os.environ.get("RANK", 0)), int(os.environ.get("WORLD_SIZE", 1))
    local = int(os.environ.get("LOCAL_RANK", 0))
    if world < 2:
        raise SystemExit("bench_shard_detect.py runs under torchrun with two or more ranks")
    from bench import MULTI_KW, multi_frames
    frames = cls = None
    if rank == 0:                                        # rendered before CUDA / NCCL exist in this process (the renderer forks)
        frames, cls = multi_frames(8, a.frames)
    import torch
    import torch.distributed as dist
    if torch.cuda.device_count() < world:
        raise SystemExit(f"{world} ranks need {world} GPUs, {torch.cuda.device_count()} visible")
    torch.cuda.set_device(local)
    dist.init_process_group("nccl", device_id=torch.device("cuda", local), timeout=datetime.timedelta(minutes=20))
    import maskfusion_b200 as mfb
    from maskfusion_b200.sharding import ShardedMaskFusion
    from scripts.bench_detect_frame import leg as single_leg, make_detector
    from scripts.bench_rpn import gpu_info
    det_rank = world - 1
    stream = torch.cuda.Stream()
    torch.cuda.set_stream(stream)
    dev = None
    if rank == 0:
        dev = [(torch.from_numpy(f[0]).cuda(), torch.from_numpy(f[1]).cuda(), torch.from_numpy(np.ascontiguousarray(f[2])).cuda()) for f in frames]
        clsp = np.ascontiguousarray(cls, np.int32)
    nets = make_detector(1024) if rank in (0, det_rank) else None
    torch.cuda.synchronize()
    n = a.frames

    def shard_leg(k):
        smf = ShardedMaskFusion(mfb.default_config(W, H, **MULTI_KW), device=local)
        if k:
            smf.attachDetector(nets[3] if rank == det_rank else None, k, det_rank)

        def run(lo, hi):
            for t in range(lo, hi):
                if rank != 0:
                    smf.processFramePtr(0, 0, 0, 0, 0, 0, False)
                elif k:
                    smf.processFramePtr(dev[t][0].data_ptr(), dev[t][1].data_ptr(), t * 33333, 0, 0, 0, True)
                else:
                    smf.processFramePtr(dev[t][0].data_ptr(), dev[t][1].data_ptr(), t * 33333, dev[t][2].data_ptr(), clsp.ctypes.data, len(clsp), True)
        run(0, a.timed_from)
        smf.mf.sync(); dist.barrier(); torch.cuda.synchronize()
        s0 = smf.stats()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record(smf.stream)
        run(a.timed_from, n)
        e1.record(smf.stream)
        smf.mf.sync(); dist.barrier(); torch.cuda.synchronize()
        s1 = smf.stats()
        ms = torch.tensor([e0.elapsed_time(e1)], device="cuda", dtype=torch.float64)
        dist.all_reduce(ms, op=dist.ReduceOp.MAX)
        ms = float(ms[0]) / (n - a.timed_from)
        owners = [smf.owner(i) for i in range(len(smf.models()))]
        if k:
            smf.detachDetector()
        smf.close()
        return {"ms_per_frame": round(ms, 4), "models": len(owners), "owners": owners,
                "nccl_calls_per_frame": round((s1["calls"] - s0["calls"]) / (n - a.timed_from), 3),
                "nccl_bytes_per_frame": round((s1["bytes"] - s0["bytes"]) / (n - a.timed_from), 1)}

    runs = {name: [] for name, _ in SHARD_LEGS + SINGLE_LEGS}
    for rep in range(a.repeats):
        order = SHARD_LEGS + SINGLE_LEGS
        for name, k in (order if rep % 2 == 0 else order[::-1]):
            if name.startswith("shard"):
                runs[name].append(shard_leg(k))
            else:
                if rank == 0:
                    runs[name].append(single_leg(stream, dev, cls, a.timed_from, nets[3], k))
                dist.barrier()
    if rank == 0:
        gpu, limit = gpu_info()
        out = {"gpu": gpu, "power_limit": limit, "n_gpus": world, "detector_rank": det_rank, "frames_timed": n - a.timed_from,
               "repeats": a.repeats, "legs": {}}
        for name, _ in SHARD_LEGS + SINGLE_LEGS:
            rs = runs[name]
            ms = [r["ms_per_frame"] for r in rs]
            e = {"ms_per_frame": round(float(np.mean(ms)), 4), "frames_per_s": round(1e3 / float(np.mean(ms)), 2), "spread_ms": [min(ms), max(ms)],
                 "models": [r["models"] for r in rs]}
            if name.startswith("shard"):
                e["owners"] = rs[-1]["owners"]
                e["nccl_calls_per_frame"] = rs[-1]["nccl_calls_per_frame"]; e["nccl_bytes_per_frame"] = rs[-1]["nccl_bytes_per_frame"]
            out["legs"][name] = e
        print(json.dumps(out))
    if nets is not None:
        nets[3].close(); nets[2].close(); nets[1].close()
    dist.destroy_process_group()


if __name__ == "__main__":
    main()
