#!/usr/bin/env python
"""Region-proposal stage and detection-head timing (csrc/mf_rpn.cu, csrc/mf_heads.cu) at 1024x1024 with synthetic weights, on a
synthetic 640x480 frame moulded by mf_backbone_mold.  CUDA-event times per stage, each averaged over --iters back-to-back launches after a warm-up:
  backbone       ResNet-101-FPN forward
  rpn_conv       shared 3x3 256->512 conv on P2..P6, with TFLOP/s and its share of the H100 SXM data-sheet dense BF16 figure (989 TFLOP/s)
  rpn_heads      the 1x1 logit + delta heads (one GEMM, fp32 output) and the split into logits / deltas
  proposals      top-6000, decode, NMS -> 1000 proposals
  roi_align      7x7 ROI Align of the 1000 proposals, with GB/s of the bytes it must move (4 bf16 corners per sample and channel + the output)
  classifier     detection heads (csrc/mf_heads.cu): FC1 (7x7 conv as one GEMM, K = 12 544), FC2, class + delta heads (fp32)
  detections     softmax, refinement, per-class NMS, top 100
  mask_head      14x14 ROI Align of the 100 detection rows, 4 x 3x3 conv (im2col + GEMM), transposed conv, mask logits, own-class sigmoid
  id_image       unmould + generate_id_image of the 640x480 frame
FC1 and the four mask convs also get kernel times from a torch.profiler run of their own (GEMM launches in stage order), with TFLOP/s and
the share of the H100 SXM data-sheet dense BF16 figure.
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


def gemm_kernel_ms(fn, per_call, iters):
    """mean device time of the k-th GEMM launch of fn (k < per_call), from a torch.profiler run of its own"""
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(iters):
            fn()
        torch.cuda.synchronize()
    ev = sorted((e for e in prof.events() if e.device_type.name == "CUDA" and "k_gemm_bf16_wgmma" in e.name), key=lambda e: e.time_range.start)
    if len(ev) != per_call * iters:
        raise RuntimeError(f"expected {per_call * iters} GEMM kernels in the trace, found {len(ev)}")
    return [sum(ev[i * per_call + k].time_range.elapsed_us() for i in range(iters)) / iters / 1000.0 for k in range(per_call)]


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
    det = mfb.Detector(rpn, seed=13)
    D = mfb.Detector
    for _ in range(warm):
        det.forward(640, 480)
    torch.cuda.synchronize()
    ms.update({
        "classifier": timed(lambda: det.run(D.CLASSIFIER), iters, st),
        "detections": timed(lambda: det.run(D.DETECTIONS), iters, st),
        "mask_head": timed(lambda: det.run(D.MASKS), iters, st),
        "id_image": timed(lambda: det.run(D.ID_IMAGE), iters, st),
    })
    gemm_ms = gemm_kernel_ms(lambda: det.run(D.CLASSIFIER | D.MASKS), 9, 10)      # FC1, FC2, heads, 4 mask convs, transposed conv, mask logits
    n_det, _ = det.detections()
    kept, _ = rpn.proposals()
    pixels = sum((S >> l) ** 2 for l in range(2, 7))
    conv_flop = 2.0 * 9 * 256 * 512 * pixels
    roi_bytes = R.POST_NMS * R.POOL * R.POOL * R.CHANNELS * 2 * (4 + 1)
    rpn_ms = ms["rpn_conv"] + ms["rpn_heads"] + ms["proposals"] + ms["roi_align"]
    heads_ms = ms["classifier"] + ms["detections"] + ms["mask_head"] + ms["id_image"]
    fc1_flop = 2.0 * 1000 * 12544 * 1024
    mconv_flop = 4 * 2.0 * 100 * 196 * 2304 * 256
    mconv_ms = sum(gemm_ms[3:7])
    name, limit = gpu_info()
    out = {
        "gpu": name, "power_limit": limit, "input": S, "anchors": rpn.A, "kept": kept, "iters": iters,
        "ms": {k: round(v, 4) for k, v in ms.items()},
        "rpn_total_ms": round(rpn_ms, 4), "rpn_over_backbone": round(rpn_ms / ms["backbone"], 4),
        "rpn_conv_gflop": round(conv_flop / 1e9, 2), "rpn_conv_tflops": round(conv_flop / ms["rpn_conv"] / 1e9, 2),
        "rpn_conv_frac_of_datasheet_bf16": round(conv_flop / ms["rpn_conv"] / 1e9 / BF16_DATASHEET_TFLOPS, 4),
        "backbone_gflop": round(bb.flops() / 1e9, 2), "backbone_tflops": round(bb.flops() / ms["backbone"] / 1e9, 2),
        "roi_align_gbps": round(roi_bytes / ms["roi_align"] / 1e6, 1),
        "n_detections": n_det, "heads_total_ms": round(heads_ms, 4),
        "fc1_gflop": round(fc1_flop / 1e9, 2), "fc1_kernel_ms": round(gemm_ms[0], 4), "fc1_tflops": round(fc1_flop / gemm_ms[0] / 1e9, 2),
        "fc1_frac_of_datasheet_bf16": round(fc1_flop / gemm_ms[0] / 1e9 / BF16_DATASHEET_TFLOPS, 4),
        "mask_convs_gflop": round(mconv_flop / 1e9, 2), "mask_convs_kernel_ms": round(mconv_ms, 4),
        "mask_convs_tflops": round(mconv_flop / mconv_ms / 1e9, 2),
        "mask_convs_frac_of_datasheet_bf16": round(mconv_flop / mconv_ms / 1e9 / BF16_DATASHEET_TFLOPS, 4),
    }
    det.close()
    rpn.close()
    bb.close()
    return out


if __name__ == "__main__":
    ap = argparse.ArgumentParser()
    ap.add_argument("--size", type=int, default=1024)
    ap.add_argument("--iters", type=int, default=50)
    a = ap.parse_args()
    print(json.dumps(run(a.size, a.iters)))
