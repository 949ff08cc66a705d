#!/usr/bin/env python
"""Frame queue (mf_set_frame_queue, the reference's -frameQ) with the on-GPU Mask R-CNN detector attached.

bench.py's configs[2] setup (single_process_multi), as scripts/bench_detect_frame.py: the table scene with 3 objects, MULTI_KW, 640x480,
device-resident inputs.  Calls [0, --timed-from) are warm-up (--timed-from must exceed the longest queue, so every timed call processes a
frame), then CUDA events around calls [--timed-from, --frames), with no synchronisation between the two: the timed window starts and ends
in the steady state of the queue.  Legs:
  masks            the scene's masks + classes as inputs, no queue
  q{L}_k{k}        detector at S = 1024 attached, every_k k, queue length L (0 = no queue), no masks given
Per leg: ms per processed frame, frames/s and the model count.  The legs run --repeats times, in alternating order; the spread over the
repeats is printed.  One JSON object, with the GPU name, power limit and SM clock read in the same run."""
import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import numpy as np
import torch
import maskfusion_b200 as mfb
from bench import MULTI_KW, multi_frames
from scripts.bench_rpn import gpu_info
from scripts.bench_detect_frame import make_detector

W, H = 640, 480
QUEUES = (0, 2, 8, 30)
LEGS = [("masks", 0, 0)] + [(f"q{q}_k{k}", q, k) for k in (1, 5) for q in QUEUES]


def sm_clock():
    """current SM clock in MHz as nvidia-smi reports it (read-only query)"""
    try:
        r = subprocess.run(["nvidia-smi", "--query-gpu=clocks.sm", "--format=csv,noheader"], capture_output=True, text=True, timeout=60)
        return r.stdout.strip().splitlines()[0] if r.stdout.strip() else None
    except (OSError, subprocess.SubprocessError):
        return None


def leg(stream, dev, cls, timed_from, det=None, queue=0, every_k=0):
    mf = mfb.MaskFusion(mfb.default_config(W, H, **MULTI_KW), stream=stream.cuda_stream)
    mf.setFrameQueue(queue)
    if det is not None:
        mf.attachDetector(det, every_k)
    else:
        mf.setFrameClasses(cls)
    torch.cuda.synchronize()

    def run(lo, hi):
        for t in range(lo, hi):
            mf.processFramePtr(dev[t][0].data_ptr(), dev[t][1].data_ptr(), t * 33333, True, mask_ptr=0 if det is not None else dev[t][2].data_ptr())
    # Steady state at both ends of the window: nothing is drained between the warm-up and the timed calls.  A synchronisation there would
    # let the network finish the detections of the queued frames before e0 while e1 does not wait for those of the frames queued at the
    # end, which favours deep queues.  Without it the network is the same number of frames ahead at e0 and at e1.
    run(0, timed_from)
    tick0 = mf.getTick()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record(stream)
    run(timed_from, len(dev))
    e1.record(stream)
    mf.sync(); torch.cuda.synchronize()
    processed = mf.getTick() - tick0
    assert processed == len(dev) - timed_from, (processed, queue)
    ms = e0.elapsed_time(e1) / processed
    models = len(mf.getModels())
    if det is not None:
        mf.attachDetector(None)
    mf.close()
    return {"ms_per_frame": round(ms, 4), "frames_per_s": round(1e3 / ms, 2), "models": models}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", type=int, default=120)
    ap.add_argument("--timed-from", type=int, default=40)
    ap.add_argument("--repeats", type=int, default=2)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_frame_queue.py measures on the GPU; no CUDA device here")
    if a.timed_from <= max(QUEUES):
        raise SystemExit(f"--timed-from must exceed the longest queue ({max(QUEUES)})")
    frames, cls = multi_frames(3, a.frames)
    dev = [(torch.from_numpy(f[0]).cuda(), torch.from_numpy(f[1]).cuda(), torch.from_numpy(np.ascontiguousarray(f[2])).cuda()) for f in frames]
    stream = torch.cuda.Stream()
    net = make_detector(1024)
    torch.cuda.synchronize()
    clocks = [sm_clock()]
    runs = {name: [] for name, _, _ in LEGS}
    for rep in range(a.repeats):
        order = LEGS if rep % 2 == 0 else LEGS[::-1]
        for name, q, k in order:
            runs[name].append(leg(stream, dev, cls, a.timed_from, net[3] if k else None, q, k))
        clocks.append(sm_clock())
    name, limit = gpu_info()
    out = {"gpu": name, "power_limit": limit, "sm_clock": clocks, "frames_timed": a.frames - a.timed_from, "repeats": a.repeats, "legs": {}}
    for lname, q, k in LEGS:
        ms = [r["ms_per_frame"] for r in runs[lname]]
        out["legs"][lname] = {"ms_per_frame": round(float(np.mean(ms)), 4), "frames_per_s": round(1e3 / float(np.mean(ms)), 2),
                              "spread_ms": [min(ms), max(ms)], "models": [r["models"] for r in runs[lname]]}
    print(json.dumps(out))
    st, bb, rpn, det = net
    det.close(); rpn.close(); bb.close()


if __name__ == "__main__":
    main()
