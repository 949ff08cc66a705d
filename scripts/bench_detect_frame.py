#!/usr/bin/env python
"""Multi-model frames with the on-GPU Mask R-CNN detector attached (mf_attach_detector) against masks as inputs.

bench.py's configs[2] setup (single_process_multi): the table scene with 3 objects, MULTI_KW, 640x480, device-resident inputs, frames
[0, --timed-from) as warm-up, then CUDA events around frames [--timed-from, --frames).  Legs:
  masks            the scene's masks + classes as inputs (the reference's -maskdir mode, today's bench path)
  det1024_k1/_k5   detector at S = 1024 attached, every_k 1 and 5, no masks given
  det256_k1        detector at S = 256, every_k 1
  detect_S         the detector's own mould + backbone + RPN + heads on one 640x480 frame, averaged over --detect-iters launches
Per leg: frames/s, ms per frame and the model count (detector masks spawn other models than the scene's masks: the workloads differ).  For
the attached legs, the share of the detection time hidden behind the dense pipeline: (ms_masks + ms_detect/k - ms_attached) / (ms_detect/k).
The legs run --repeats times, in alternating order; the spread over the repeats is printed.  One JSON object, with the GPU name and power
limit read in the same run."""
import argparse
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import numpy as np
import torch
import maskfusion_b200 as mfb
from bench import MULTI_KW, multi_frames
from scripts.bench_rpn import gpu_info

W, H = 640, 480
LEGS = [("masks", 0, 0), ("det1024_k1", 1024, 1), ("det1024_k5", 1024, 5), ("det256_k1", 256, 1)]


def make_detector(S):
    st = torch.cuda.Stream()
    bb = mfb.Backbone(S, seed=7, stream=st.cuda_stream)
    rpn = mfb.RegionProposals(bb, seed=11)
    det = mfb.Detector(rpn, seed=13)
    return st, bb, rpn, det


def leg(stream, dev, cls, timed_from, det=None, every_k=0):
    mf = mfb.MaskFusion(mfb.default_config(W, H, **MULTI_KW), stream=stream.cuda_stream)
    if det is not None:
        mf.attachDetector(det, every_k)
    else:
        mf.setFrameClasses(cls)
    torch.cuda.synchronize()

    def run(lo, hi):
        for t in range(lo, hi):
            mf.processFramePtr(dev[t][0].data_ptr(), dev[t][1].data_ptr(), t * 33333, True, mask_ptr=0 if det is not None else dev[t][2].data_ptr())
    run(0, timed_from)
    mf.sync(); torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record(stream)
    run(timed_from, len(dev))
    e1.record(stream)
    mf.sync(); torch.cuda.synchronize()
    ms = e0.elapsed_time(e1) / (len(dev) - timed_from)
    models = len(mf.getModels())
    if det is not None:
        mf.attachDetector(None)
    mf.close()
    return {"ms_per_frame": round(ms, 4), "frames_per_s": round(1e3 / ms, 2), "models": models}


def detect_ms(det, rgba, iters, st):
    for _ in range(3):
        det.detect(rgba.data_ptr(), W, H)
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record(st)
    for _ in range(iters):
        det.detect(rgba.data_ptr(), W, H)
    e1.record(st)
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / iters


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", type=int, default=60)
    ap.add_argument("--timed-from", type=int, default=20)
    ap.add_argument("--repeats", type=int, default=2)
    ap.add_argument("--detect-iters", type=int, default=50)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_detect_frame.py measures on the GPU; no CUDA device here")
    frames, cls = multi_frames(3, a.frames)
    dev = [(torch.from_numpy(f[0]).cuda(), torch.from_numpy(f[1]).cuda(), torch.from_numpy(np.ascontiguousarray(f[2])).cuda()) for f in frames]
    rgba = torch.from_numpy(np.concatenate([frames[a.timed_from][0], np.full((H, W, 1), 255, np.uint8)], axis=2)).cuda()
    stream = torch.cuda.Stream()
    nets = {S: make_detector(S) for S in (256, 1024)}
    torch.cuda.synchronize()
    runs = {name: [] for name, _, _ in LEGS}
    det_runs = {S: [] for S in nets}
    for rep in range(a.repeats):
        order = LEGS if rep % 2 == 0 else LEGS[::-1]
        for name, S, k in order:
            runs[name].append(leg(stream, dev, cls, a.timed_from, nets[S][3] if S else None, k))
        for S in (sorted(nets) if rep % 2 == 0 else sorted(nets, reverse=True)):
            det_runs[S].append(detect_ms(nets[S][3], rgba, a.detect_iters, nets[S][0]))
    name, limit = gpu_info()
    out = {"gpu": name, "power_limit": limit, "frames_timed": a.frames - a.timed_from, "repeats": a.repeats, "legs": {}}
    for S, v in det_runs.items():
        out["legs"][f"detect_{S}"] = {"ms_per_detect": round(float(np.mean(v)), 4), "runs": [round(x, 4) for x in v]}
    ms_masks = float(np.mean([r["ms_per_frame"] for r in runs["masks"]]))
    for lname, S, k in LEGS:
        rs = runs[lname]
        ms = [r["ms_per_frame"] for r in rs]
        e = {"ms_per_frame": round(float(np.mean(ms)), 4), "frames_per_s": round(1e3 / float(np.mean(ms)), 2), "spread_ms": [min(ms), max(ms)],
             "models": [r["models"] for r in rs]}
        if S:
            dk = float(np.mean(det_runs[S])) / k
            e["hidden_fraction"] = round((ms_masks + dk - float(np.mean(ms))) / dk, 4)
        out["legs"][lname] = e
    print(json.dumps(out))
    for st, bb, rpn, det in nets.values():
        det.close(); rpn.close(); bb.close()


if __name__ == "__main__":
    main()
