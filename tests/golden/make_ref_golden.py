"""Writes tests/golden/ref_kernels_golden.npz: the reference's own CUDA kernels (oracle/_ref/libmf_ref.so, oracle/Makefile.ref) run on the
inputs tests/test_gpu_ref.py builds from the CPU oracle.  Needs a GPU.  Maps are stored as validity masks plus seeded pixel samples.

    python tests/golden/make_ref_golden.py [OUT.npz]
"""
from __future__ import annotations

import ctypes as C
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)

from tests import oracle_lib as ol                         # noqa: E402
from tests import test_gpu_ref as T                        # noqa: E402

f32p = C.POINTER(C.c_float)
W, H = T.W, T.H


def main(out_path):
    ref = C.CDLL(os.path.join(ROOT, "oracle", "_ref", "libmf_ref.so"))
    sc, orc, pose_before = T.make_state()
    fa = orc.frame_arrays(); od = orc.odom(0)
    g = {}
    idx = [T.sample_index(l) for l in range(3)]
    for l in range(3):
        g[f"idx{l}"] = idx[l]
    g["idxw"] = idxw = T.sample_index(0, T.N_SAMPLE_IMG, seed=200)

    def put_map(name, a, l):
        g[name + "_nan"] = np.packbits(np.isnan(a[0]).ravel())
        g[name + "_val"] = a.reshape(3, -1)[:, idx[l]]

    # vertex / normal maps of the frame pyramid (cudafuncs.cu createVMap / createNMap)
    for l in range(3):
        w, h = W >> l, H >> l
        v = np.zeros((3, h, w), np.float32); n = np.zeros((3, h, w), np.float32)
        d = np.ascontiguousarray(fa[f"depth{l}"])
        assert ref.ref_vmap_nmap(ol.ptr(d), w, h, C.c_float(528 / (1 << l)), C.c_float(528 / (1 << l)), C.c_float(320 / (1 << l)),
                                 C.c_float(240 / (1 << l)), C.c_float(4.0), ol.ptr(v), ol.ptr(n)) == 0
        put_map(f"vmap{l}", v, l); put_map(f"nmap{l}", n, l)
    # depth pyramid (pyrDown) and the Gaussian u8 pyramid on a seeded image
    for l in range(2):
        w, h = W >> l, H >> l
        out = np.zeros((h // 2, w // 2), np.float32)
        assert ref.ref_pyrdown_f(ol.ptr(np.ascontiguousarray(fa[f"depth{l}"])), w, h, ol.ptr(out)) == 0
        g[f"pyrf{l}_val"] = out.ravel()[idx[l + 1]]
    src = T.pyr_u8_input()
    o1 = np.zeros((H // 2, W // 2), np.uint8)
    assert ref.ref_pyrdown_u8(ol.ptr(src), W, H, ol.ptr(o1)) == 0
    g["pyru8"] = o1
    # model maps (predicted vertex / normal maps in the model frame)
    m = orc.p.model(0)
    fill = bool(orc.L.orc_requires_fill_in(m.splatImage, W, H, C.c_float(0.75)))
    vt = np.ascontiguousarray(orc.p.tex(0, "fillVertex" if fill else "splatVertex"))
    nt = np.ascontiguousarray(orc.p.tex(0, "fillNormal" if fill else "splatNormal"))
    vs = [np.zeros((3, H >> l, W >> l), np.float32) for l in range(3)]
    ns = [np.zeros((3, H >> l, W >> l), np.float32) for l in range(3)]
    vp = (f32p * 3)(*[a.ctypes.data_as(f32p) for a in vs]); npp = (f32p * 3)(*[a.ctypes.data_as(f32p) for a in ns])
    R = np.ascontiguousarray(pose_before[:3, :3]); t = np.ascontiguousarray(pose_before[:3, 3])
    assert ref.ref_model_maps(ol.ptr(vt), ol.ptr(nt), W, H, ol.ptr(R), ol.ptr(t), vp, npp) == 0
    for l in range(3):
        put_map(f"mvmap{l}", vs[l], l); put_map(f"mnmap{l}", ns[l], l)
    # icpStep with the reference's fallback launch config 128x112
    P = pose_before
    Rpi = np.ascontiguousarray(np.linalg.inv(P[:3, :3].astype(np.float64)).astype(np.float32))
    Rc = np.ascontiguousarray(P[:3, :3]); tc = np.ascontiguousarray(P[:3, 3])
    for l in range(3):
        w, h = W >> l, H >> l
        A = np.zeros(36, np.float32); b = np.zeros(6, np.float32); res = np.zeros(2, np.float32)
        vg = ol.arr(od.vmap_g[l], (3, h, w), np.float32); ng = ol.arr(od.nmap_g[l], (3, h, w), np.float32)
        assert ref.ref_icp_step(ol.ptr(Rc), ol.ptr(tc), ol.ptr(fa[f"vmap{l}"]), ol.ptr(fa[f"nmap{l}"]), ol.ptr(Rpi), ol.ptr(tc),
                                C.c_float(528 / (1 << l)), C.c_float(528 / (1 << l)), C.c_float(320 / (1 << l)), C.c_float(240 / (1 << l)),
                                ol.ptr(np.ascontiguousarray(vg)), ol.ptr(np.ascontiguousarray(ng)), C.c_float(0.1),
                                C.c_float(np.float32(np.sin(20.0 * 3.14159254 / 180.0))), w, h, 128, 112, ol.ptr(A), ol.ptr(b), ol.ptr(res)) == 0
        g[f"icp{l}_A"], g[f"icp{l}_b"], g[f"icp{l}_res"] = A, b, res
    # Sobel and one SO(3) step
    inten, a, b2 = T.sobel_so3_inputs(sc, orc)
    dx = np.zeros((H, W), np.int16); dy = np.zeros((H, W), np.int16)
    assert ref.ref_sobel(ol.ptr(inten), W, H, ol.ptr(dx), ol.ptr(dy)) == 0
    g["sobel_dx"] = dx.ravel()[idxw]; g["sobel_dy"] = dy.ravel()[idxw]
    basis, kinv, krlr = T.so3_matrices()
    A = np.zeros(9, np.float32); bb = np.zeros(3, np.float32); res = np.zeros(2, np.float32)
    assert ref.ref_so3_step(ol.ptr(a), ol.ptr(b2), ol.ptr(basis), ol.ptr(kinv), ol.ptr(krlr), W // 4, H // 4, 160, 64, ol.ptr(A), ol.ptr(bb), ol.ptr(res)) == 0
    g["so3_A"], g["so3_b"], g["so3_res"] = A, bb, res
    # geometric edges (segmentation.cu)
    e = np.zeros((H, W), np.float32); inv = np.zeros((H, W), np.uint8)
    assert ref.ref_geometric_edges(ol.ptr(fa["vmap0"]), ol.ptr(fa["nmap0"]), W, H, C.c_float(150.0), C.c_float(2.8), C.c_float(0.3), ol.ptr(e), ol.ptr(inv)) == 0
    g["edges_val"] = e.ravel()[idxw]; g["edges_inv"] = inv
    # computeRgbResidual + projectToPointCloud + rgbStep, one iteration per level on the oracle's odometry state
    for l in range(3):
        w, h = W >> l, H >> l
        x = T.rgb_level_inputs(orc, l)
        cnt_r, sig_r = C.c_int(0), C.c_int(0)
        A = np.zeros(36, np.float32); b = np.zeros(6, np.float32)
        fx, fy, cx, cy = x["cam"]
        rc = ref.ref_rgb_iteration(C.c_float(x["minScale"]), ol.ptr(x["gx"]), ol.ptr(x["gy"]), ol.ptr(x["ld"]), ol.ptr(x["nd"]), ol.ptr(x["li"]), ol.ptr(x["ni"]),
                                   C.c_float(0.07), ol.ptr(x["kt"]), ol.ptr(x["krk"]), C.c_float(float(x["cnt_o"])), C.c_float(fx), C.c_float(fy),
                                   C.c_float(cx), C.c_float(cy), l, C.c_float(x["sobelScale"]), w, h, C.byref(cnt_r), C.byref(sig_r), ol.ptr(A), ol.ptr(b))
        assert rc == 0
        g[f"rgb{l}_cnt"] = np.int64(cnt_r.value); g[f"rgb{l}_sig"] = np.int64(sig_r.value); g[f"rgb{l}_A"] = A; g[f"rgb{l}_b"] = b
    np.savez_compressed(out_path, **g)
    print(out_path, os.path.getsize(out_path), "bytes")


if __name__ == "__main__":
    main(sys.argv[1] if len(sys.argv) > 1 else os.path.join(ROOT, "tests", "golden", "ref_kernels_golden.npz"))
