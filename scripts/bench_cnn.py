#!/usr/bin/env python
"""Backbone (ResNet-101-FPN, 1024x1024, synthetic weights) timing: tensor-pipe utilisation of the wgmma GEMMs.
Prints one JSON object; used by bench.py (key "backbone")."""
import json, os, sys, time
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
import maskfusion_b200 as mfb

def run(S=1024, iters=10, warm=3, per_layer=False):
    st = torch.cuda.current_stream()
    bb = mfb.Backbone(S, seed=3, stream=st.cuda_stream)
    x = (torch.randn(S, S, 3, device="cuda") * 60).to(torch.bfloat16).contiguous()
    for _ in range(warm):
        bb.forward(x.data_ptr())
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record(st)
    for _ in range(iters):
        bb.forward(x.data_ptr())
    e1.record(st)
    torch.cuda.synchronize()
    ms = e0.elapsed_time(e1) / iters
    fl = bb.flops()
    peaks = json.load(open(os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "MEASURED_PEAKS.json"))) if os.path.exists(os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "MEASURED_PEAKS.json")) else {"bf16_tflops": 989.0}      # H100 SXM data sheet, dense BF16, 700 W part
    out = {"input": S, "gemms": bb.numGemms(), "gflop": round(fl / 1e9, 2), "ms": round(ms, 4), "tflops": round(fl / ms / 1e9, 2),
           "peak_tflops_burst": peaks["bf16_tflops"], "frac_of_burst_peak": round(fl / ms / 1e9 / peaks["bf16_tflops"], 4)}
    # cuDNN/torch bf16 channels_last conv forward of the same layer stack = library comparison point (BASELINE.md B-cnn)
    bb.close()
    return out

if __name__ == "__main__":
    S = int(sys.argv[1]) if len(sys.argv) > 1 else 1024
    print(json.dumps(run(S, iters=int(sys.argv[2]) if len(sys.argv) > 2 else 10)))
