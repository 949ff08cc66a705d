#!/usr/bin/env python
"""Stage clock of k_track_persistent (profiling build: MFB200_TAG=timing MFB200_DEFINES=-DMF_TRACK_TIMING python -m maskfusion_b200.build):
per pyramid level, the average time CTA 0 spends in each stage of a reduction step.

    MFB200_TAG=timing python scripts/track_timing.py [--bench-state] [--frames F] [--avg A]

clock64 counts SM cycles; they are converted with the median SM clock NVML reports while the frames run (printed as sm_mhz).
--bench-state tracks the state bench.py times: the -static configuration with the background store pre-populated to ~4.7 M surfels.
Without it, a 700 k-surfel store that holds only what the frames fuse.  The stages are averaged over the last A tracking launches."""
import argparse
import collections
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
os.environ.setdefault("MFB200_TAG", "timing")


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--bench-state", action="store_true", help="bench.py's configs[1] state: 4.7 M pre-populated surfels")
    ap.add_argument("--frames", type=int, default=16)
    ap.add_argument("--avg", type=int, default=8, help="launches (the last ones) the stages are averaged over")
    args = ap.parse_args()
    import bench
    import maskfusion_b200 as mfb
    from maskfusion_b200.synth import SynthScene
    W, H = 640, 480
    sc = SynthScene(W, H, n_objects=0, seed=0)
    mf = mfb.MaskFusion(mfb.default_config(W, H, capacityGlobal=bench.CAPACITY if args.bench_state else 700000))
    rgb, depth, *_ = sc.render(0)
    mf.processFrame(rgb, depth, 0)
    if args.bench_state:
        bench.prepopulate(mf, sc)
    sampler = bench.ClockSampler(0)
    sampler.start()
    runs = []
    buf = np.zeros(8192, np.int64)
    for t in range(1, args.frames + 1):
        rgb, depth, *_ = sc.render(t)
        mf.processFrame(rgb, depth, t * 33333)
        if t > args.frames - args.avg:
            n = mf.L.mf_debug_track_timing(buf.ctypes.data, 8192)          # synchronises the device
            runs.append(buf[:n].reshape(-1, 2).copy())
    mf.sync()
    clocks = sampler.stop()
    if not clocks.get("sm_mhz"):
        raise SystemExit("no SM clock from NVML: cycles cannot be converted to time (%s)" % clocks["reasons"])
    ghz = clocks["sm_mhz"] / 1e3
    names = {2: "A pixels", 5: "A reduce+exchange+sum", 6: "B pixels (+sigma)", 9: "B reduce+exchange+sum", 20: "solve: assemble A, b", 21: "solve: pivoted LDLT", 22: "solve: rodrigues", 23: "solve: pose composition", 10: "solve: warp constants + barrier",
             12: "so3 pixels", 15: "so3 reduce+exchange+sum", 16: "so3 solve"}
    acc = collections.defaultdict(lambda: [0, 0.0])
    total = 0.0
    for ev in runs:
        level = "so3"
        prev = None
        for tag, clk in ev:
            tag = int(tag)
            if tag in (100, 101, 102):
                level = f"L{tag - 100}"
            if tag == 11:
                level = "so3"
            if prev is not None and tag in names:
                a = acc[(level, names[tag])]; a[0] += 1; a[1] += (clk - prev) / ghz / 1e3
            prev = clk
        total += float(ev[-1, 1] - ev[0, 1]) / ghz / 1e3
    out = {"sm_mhz": clocks["sm_mhz"], "sm_max_mhz": clocks["sm_max_mhz"], "clock_reasons": clocks["reasons"], "bench_state": args.bench_state,
           "launches": len(runs), "total_us": round(total / len(runs), 1), "stages_us": {}}
    for (lv, nm), (c, us) in sorted(acc.items()):
        out["stages_us"].setdefault(lv, {})[nm] = {"n_per_launch": round(c / len(runs), 2), "avg_us": round(us / c, 2), "total_us": round(us / len(runs), 1)}
    mf.close()
    print(json.dumps(out, indent=1))


if __name__ == "__main__":
    main()
