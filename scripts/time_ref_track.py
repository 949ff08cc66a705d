#!/usr/bin/env python
"""B-ref-cuda (SURVEY 8d-iii): the REFERENCE's own CUDA kernels (reduce.cu / cudafuncs.cu compiled unmodified into
oracle/_ref/libmf_ref.so) timed on this GPU for one model-frame of tracking in the reference's calling pattern -- model-map
preparation, photometric pyramids, SO(3) pre-alignment, 4/5/10 x (computeRgbResidual + icpStep + rgbStep), each call with its own
launches, device synchronisations, allocations and D2H copies (oracle/ref_shim/ref_api.cu: ref_track_schedule_time_ms).
The GL half of the reference (surfel passes) cannot run here.  Test infrastructure; bench.py imports run()."""
import ctypes as C
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def run(reps=10):
    from tests import oracle_lib as ol
    from tests.stagewise import OracleStages
    from maskfusion_b200.synth import SynthScene
    path = os.path.join(ROOT, "oracle", "_ref", "libmf_ref.so")
    if not os.path.exists(path):
        return {"unavailable": "oracle/_ref/libmf_ref.so not built (needs /root/reference at build time)"}
    ref = C.CDLL(path)
    W, H = 640, 480
    sc = SynthScene(W, H, n_objects=0, seed=0)
    orc = OracleStages(ol.default_config(W, H, capacityGlobal=600000))
    for t in range(2):
        rgb, depth, *_ = sc.render(t)
        orc.p.process_frame(rgb, depth, t)
    rgb, depth, *_ = sc.render(2)
    P = orc.pose(0).copy()
    orc.set_frame(rgb, depth); orc.generate_maps()
    fa = orc.frame_arrays()
    vtex = np.ascontiguousarray(orc.p.tex(0, "splatVertex")); ntex = np.ascontiguousarray(orc.p.tex(0, "splatNormal"))
    inten = np.zeros((H, W), np.uint8); last = np.zeros((H, W), np.uint8)
    orc.L.orc_rgb_to_intensity(ol.ptr(np.ascontiguousarray(rgb)), W, H, ol.ptr(inten))
    orc.L.orc_rgb_to_intensity(ol.ptr(np.ascontiguousarray(sc.render(1)[0])), W, H, ol.ptr(last))
    vm = (C.c_void_p * 3)(*[ol.ptr(fa[f"vmap{l}"]) for l in range(3)]); nm = (C.c_void_p * 3)(*[ol.ptr(fa[f"nmap{l}"]) for l in range(3)])
    R = np.ascontiguousarray(P[:3, :3]); t3 = np.ascontiguousarray(P[:3, 3])
    ms = np.zeros(5, np.float32)
    rc = ref.ref_track_schedule_time_ms(ol.ptr(vtex), ol.ptr(ntex), vm, nm, ol.ptr(last), ol.ptr(inten), ol.ptr(R), ol.ptr(t3),
                                        C.c_float(528.0), C.c_float(528.0), C.c_float(320.0), C.c_float(240.0), W, H, 10, int(reps), ol.ptr(ms))
    if rc != 0:
        return {"error": f"ref_track_schedule_time_ms returned {rc}"}
    return {"ref_cuda_us_per_model_frame": round(float(ms[0]) * 1e3, 1),
            "parts_us": {"model_maps": round(float(ms[1]) * 1e3, 1), "rgb_pyramids": round(float(ms[2]) * 1e3, 1),
                         "so3_10_iterations": round(float(ms[3]) * 1e3, 1), "levels_4_5_10": round(float(ms[4]) * 1e3, 1)},
            "what": "reference reduce.cu/cudafuncs.cu (unmodified, sm_90a, its own flags and launch shapes) in the calling pattern of "
                    "RGBDOdometry.cpp:153-476 on a VGA frame; host Eigen solves and the GL surfel passes not included", "reps": int(reps)}


if __name__ == "__main__":
    print(json.dumps(run()))
