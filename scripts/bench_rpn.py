#!/usr/bin/env python
"""Region-proposal stage timing (csrc/mf_rpn.cu) at 1024x1024 with synthetic weights, on a synthetic 640x480 frame moulded by
mf_backbone_mold.  CUDA-event times per stage, each averaged over --iters back-to-back launches after a warm-up:
  backbone       ResNet-101-FPN forward
  rpn_conv       shared 3x3 256->512 conv on P2..P6, with TFLOP/s and its share of the H100 SXM data-sheet dense BF16 figure (989 TFLOP/s)
  rpn_heads      the 1x1 logit + delta heads (one GEMM, fp32 output) and the split into logits / deltas
  proposals      top-6000, decode, NMS -> 1000 proposals
  roi_align      7x7 ROI Align of the 1000 proposals, with GB/s of the bytes it must move (4 bf16 corners per sample and channel + the output)
Prints one JSON object, with the GPU name and power limit read in the same run."""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np
import torch
import maskfusion_b200 as mfb
from maskfusion_b200.synth import SynthScene

BF16_DATASHEET_TFLOPS = 989.0          # H100 SXM, dense BF16, 700 W part: a data-sheet figure, not a measured peak


def gpu_info():
    props = torch.cuda.get_device_properties(0)
    limit = None
    try:
        r = subprocess.run(["nvidia-smi", "--query-gpu=uuid,power.limit", "--format=csv,noheader"], capture_output=True, text=True, timeout=60)
        rows = [l.split(", ") for l in r.stdout.strip().splitlines() if l]
        uuid = str(getattr(props, "uuid", ""))
        match = [p for u, p in rows if uuid and uuid in u]
        limit = (match or [rows[0][1]])[0] if rows else None
    except (OSError, subprocess.SubprocessError, IndexError):
        pass
    return props.name, limit


def timed(fn, iters, stream):
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record(stream)
    for _ in range(iters):
        fn()
    e1.record(stream)
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / iters


def run(S=1024, iters=50, warm=5):
    st = torch.cuda.current_stream()
    L = mfb.load_library()
    bb = mfb.Backbone(S, seed=3, stream=st.cuda_stream)
    rgb, *_ = SynthScene(640, 480, n_objects=2, seed=1).render(0)
    rgba = torch.from_numpy(np.concatenate([rgb, np.full(rgb.shape[:2] + (1,), 255, np.uint8)], axis=2)).cuda()
    if L.mf_backbone_mold(C.c_void_p(bb.h), C.c_void_p(rgba.data_ptr()), 640, 480) != 0:
        raise mfb.MFError("mold failed")
    inp = L.mf_backbone_input_buffer(bb.h)
    rpn = mfb.RegionProposals(bb, seed=11)
    R = mfb.RegionProposals
    for _ in range(warm):
        bb.forward(inp)
        rpn.forward()
    torch.cuda.synchronize()
    ms = {
        "backbone": timed(lambda: bb.forward(inp), iters, st),
        "rpn_conv": timed(lambda: rpn.run(R.CONV), iters, st),
        "rpn_heads": timed(lambda: rpn.run(R.HEADS), iters, st),
        "proposals": timed(lambda: rpn.run(R.PROPOSALS), iters, st),
        "roi_align": timed(lambda: rpn.run(R.ROI_ALIGN), iters, st),
    }
    kept, _ = rpn.proposals()
    pixels = sum((S >> l) ** 2 for l in range(2, 7))
    conv_flop = 2.0 * 9 * 256 * 512 * pixels
    roi_bytes = R.POST_NMS * R.POOL * R.POOL * R.CHANNELS * 2 * (4 + 1)
    rpn_ms = ms["rpn_conv"] + ms["rpn_heads"] + ms["proposals"] + ms["roi_align"]
    name, limit = gpu_info()
    out = {
        "gpu": name, "power_limit": limit, "input": S, "anchors": rpn.A, "kept": kept, "iters": iters,
        "ms": {k: round(v, 4) for k, v in ms.items()},
        "rpn_total_ms": round(rpn_ms, 4), "rpn_over_backbone": round(rpn_ms / ms["backbone"], 4),
        "rpn_conv_gflop": round(conv_flop / 1e9, 2), "rpn_conv_tflops": round(conv_flop / ms["rpn_conv"] / 1e9, 2),
        "rpn_conv_frac_of_datasheet_bf16": round(conv_flop / ms["rpn_conv"] / 1e9 / BF16_DATASHEET_TFLOPS, 4),
        "backbone_gflop": round(bb.flops() / 1e9, 2), "backbone_tflops": round(bb.flops() / ms["backbone"] / 1e9, 2),
        "roi_align_gbps": round(roi_bytes / ms["roi_align"] / 1e6, 1),
    }
    rpn.close()
    bb.close()
    return out


if __name__ == "__main__":
    ap = argparse.ArgumentParser()
    ap.add_argument("--size", type=int, default=1024)
    ap.add_argument("--iters", type=int, default=50)
    a = ap.parse_args()
    print(json.dumps(run(a.size, a.iters)))
