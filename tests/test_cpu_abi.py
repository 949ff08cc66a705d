"""The C ABI boundary without a device: the ctypes bindings follow include/maskfusion_b200.h, every refusal lands in the calling thread's
mf_last_error() (mf_cnn_last_error() returns the same text), and one thread's refusal never shows in another's.  The calls run in a
subprocess that sees no CUDA device and pass null pointers, as in tests/test_cpu_cnn.py."""
from __future__ import annotations

import ctypes as C
import inspect
import json
import os
import re
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HEADER = os.path.join(ROOT, "include", "maskfusion_b200.h")
SCALARS = {"int": C.c_int, "unsigned": C.c_uint, "int64_t": C.c_int64, "float": C.c_float, "double": C.c_double}


def _child(src: str, *args: str):
    env = dict(os.environ, CUDA_VISIBLE_DEVICES="")
    r = subprocess.run([sys.executable, "-c", src, *args], capture_output=True, text=True, env=env, cwd=ROOT, timeout=300)
    assert r.returncode == 0, r.stderr
    return json.loads(r.stdout.strip().splitlines()[-1])


def _expected(decl: str) -> str:
    """the name of the ctypes type a declaration (without its name) binds to"""
    t = re.sub(r"\b(const|struct)\b|\s", "", decl)
    if t == "void":
        return "None"
    if t == "char*":
        return "c_char_p"
    return "c_void_p" if t.endswith("*") else SCALARS[t].__name__           # c_int64 is c_long on LP64


def _header():
    """{name: (return type, [parameter types])} of the header's prototypes, as ctypes type names"""
    text = re.sub(r"/\*.*?\*/", "", open(HEADER).read(), flags=re.S)
    text = "\n".join(line for line in text.splitlines() if not line.lstrip().startswith("#"))
    out = {}
    for ret, name, params in re.findall(r"([\w\s*]+?)\s*\b(mf_\w+)\s*\(([^)]*)\)\s*;", text):
        types = []
        for p in params.split(","):
            p = p.strip()
            if p == "void":
                continue
            if p.endswith("]"):                                   # float pose16[16]
                types.append("c_void_p")
            else:
                types.append(_expected(p[:re.search(r"\w+$", p).start()]))
        out[name] = (_expected(ret), types)
    return out


_BINDINGS = r"""
import json
import maskfusion_b200 as mfb
L = mfb.load_library()
name = lambda t: "None" if t is None else t.__name__
print(json.dumps({n: [name(getattr(L, n).restype), [name(t) for t in getattr(L, n).argtypes]] for n in mfb.EXPORTS}))
"""


def test_ctypes_bindings_follow_the_header(product_lib):
    hdr = _header()
    assert len(hdr) == 138 and set(hdr) == set(product_lib.EXPORTS)
    # the segmentation test hook: context, 3 input images + mask count + classes, projected ids, model list, next id, allow-new, 3 outputs
    assert hdr["mf_debug_segment"] == ("c_int", ["c_void_p"] * 4 + ["c_int", "c_void_p", "c_void_p", "c_int", "c_void_p", "c_void_p", "c_int",
                                                                     "c_int", "c_void_p", "c_void_p", "c_void_p"])
    got = _child(_BINDINGS)
    for name, (ret, params) in hdr.items():
        assert got[name] == [ret, params], name
    pointers = sorted(n for n, (ret, _) in hdr.items() if ret in ("c_void_p", "c_char_p"))
    assert len(pointers) == 12, pointers
    assert [n for n in pointers if hdr[n][0] == "c_char_p"] == ["mf_cnn_last_error", "mf_last_error"]
    # the binder is the only place that sets a signature
    api = sys.modules["maskfusion_b200.api"]
    for attr in (".argtypes", ".restype"):
        assert inspect.getsource(api).count(attr) == inspect.getsource(api.load_library).count(attr) == 1, attr


_REFUSALS = r"""
import ctypes as C, json, sys
import maskfusion_b200 as mfb
L = mfb.load_library()
cfg = mfb.Config(); L.mf_config_defaults(C.byref(cfg), 640, 480)
w, h = C.c_int(0), C.c_int(0)
calls = [
    lambda: L.mf_create(C.byref(cfg), 0, None),
    lambda: L.mf_conv3x3_bf16(None, None, None, None, None, 48, 48, 64, 64, 1, None),
    lambda: L.mf_mrcnn_read_layer(sys.argv[1].encode(), b"res4x_branch2a", None, None, (C.c_int * 2)()),
    lambda: L.mf_dir_open(None, None, None, 4, b"", b"", b""),
    lambda: L.mf_klg_open(sys.argv[1].encode(), 64, 48, 0),
    lambda: L.mf_decode_jpeg(b"\x00\x01\x02\x03", 4, None, 0, C.byref(w), C.byref(h)),
]
out = []
for call in calls:
    rc = call()
    out.append([rc, L.mf_last_error().decode(), L.mf_cnn_last_error().decode()])
print(json.dumps(out))
"""


def test_every_family_reports_through_one_slot(product_lib, tmp_path):
    missing = str(tmp_path / "missing.klg")
    got = _child(_REFUSALS, missing)
    assert all(text == cnn_text for _, text, cnn_text in got), got
    rc, text, _ = got[0]                                  # the rest of the message is the CUDA runtime's own
    assert rc is None and text.startswith("no CUDA device: this library has no CPU fallback ("), text
    assert [g[:2] for g in got[1:]] == [[-2, "conv3x3: unsupported geometry"], [-1, "mrcnn_read_layer: no layer named 'res4x_branch2a'"],
                                        [None, "mf_dir_open: null colour directory"], [None, "Could not open log-file: " + missing],
                                        [-2, "not a JPEG stream"]]


_MRCNN = r"""
import ctypes as C, json
import maskfusion_b200 as mfb
L = mfb.load_library()
i6 = (C.c_int * 6)()
calls = [
    lambda: L.mf_backbone_create(100, 0, None), lambda: L.mf_rpn_create(None, 0), lambda: L.mf_detector_create(None, 0),
    lambda: L.mf_gemm_bf16(None, None, None, None, None, 0, 64, 64, 0, None),
    lambda: L.mf_backbone_num_layers(None), lambda: L.mf_backbone_get_weights(None, 0, None, None),
    lambda: L.mf_backbone_load_weights(None, b"x"), lambda: L.mf_backbone_mold(None, None, 640, 480), lambda: L.mf_backbone_forward(None, None),
    lambda: L.mf_backbone_layer(None, 0, i6), lambda: L.mf_backbone_download(None, 4, None),
    lambda: L.mf_rpn_run(None, 15), lambda: L.mf_rpn_forward(None), lambda: L.mf_rpn_propose(None, None, None, None, 1),
    lambda: L.mf_rpn_get_weights(None, None, None, None, None), lambda: L.mf_rpn_load_weights(None, b"x"), lambda: L.mf_rpn_get_anchors(None, None),
    lambda: L.mf_rpn_get_head_outputs(None, None, None), lambda: L.mf_rpn_download_conv(None, 0, None), lambda: L.mf_rpn_get_proposals(None, None),
    lambda: L.mf_rpn_get_pooled(None, None),
    lambda: L.mf_roi_align_bf16(None, None, 1, 7, None),
    lambda: L.mf_detector_run(None, 15), lambda: L.mf_detector_forward(None, 640, 480), lambda: L.mf_detector_detect(None, None, 640, 480),
    lambda: L.mf_detector_set_export(None, 0.5, None, 0, None, 0), lambda: L.mf_detector_refine(None, None, None, None, 1),
    lambda: L.mf_detector_paste(None, None, None, 640, 480), lambda: L.mf_detector_load_weights(None, b"x"),
    lambda: L.mf_detector_get_fc(None, None, None), lambda: L.mf_detector_get_head_outputs(None, None, None),
    lambda: L.mf_detector_get_mask_layer(None, 0, None), lambda: L.mf_detector_get_detections(None, None), lambda: L.mf_detector_get_masks(None, None),
    lambda: L.mf_detector_get_id_image(None, None, None, None), lambda: L.mf_detector_image_size(None, None, None),
    lambda: L.mf_detector_layer(None, 0, i6), lambda: L.mf_detector_get_weights(None, 0, None, None),
]
print(json.dumps([[call(), L.mf_last_error().decode()] for call in calls]))
"""


def test_mask_rcnn_refusals_without_a_device(product_lib):
    """every Mask R-CNN entry point that can fail, refused before device work: return code and text, as the library has always given them"""
    want = [[None, "input size must be a multiple of 64 (mrcnn: IMAGE_MAX_DIM=1024)"], [None, "rpn: no backbone"],
            [None, "detector: no region-proposal handle"], [-2, "gemm: need M > 0, and K > 0 and N > 0 multiples of 64"]]
    want += [[-1, "backbone: null handle"]] * 5 + [[-1, "backbone: bad layer index"], [-1, "backbone: no handle or level outside 0..8"]]
    want += [[-1, "rpn: null handle"]] * 10 + [[-1, "roi_align: no backbone"]]
    want += [[-1, "detector: null handle"]] * 14 + [[-1, "detector: bad layer index"]] * 2
    assert _child(_MRCNN) == want


_THREADS = r"""
import ctypes as C, json, threading
import maskfusion_b200 as mfb
L = mfb.load_library()
read = lambda: [L.mf_last_error().decode(), L.mf_cnn_last_error().decode()]
refused, b_done, seen = threading.Event(), threading.Event(), {}

def thread_a():
    seen["a_rc"] = L.mf_conv3x3_bf16(None, None, None, None, None, 48, 48, 64, 64, 1, None)
    refused.set()
    b_done.wait()
    seen["a"] = read()

def thread_b():
    refused.wait()
    seen["b_before"] = read()
    seen["b_rc"] = L.mf_mrcnn_read_layer(b"unused.safetensors", b"no_such_layer", None, None, (C.c_int * 2)())
    seen["b_after"] = read()
    b_done.set()

ts = [threading.Thread(target=thread_a), threading.Thread(target=thread_b)]
for t in ts:
    t.start()
for t in ts:
    t.join()
print(json.dumps(seen))
"""


def test_a_refusal_stays_on_its_thread(product_lib):
    a_text = "conv3x3: unsupported geometry"
    b_text = "mrcnn_read_layer: no layer named 'no_such_layer'"
    seen = _child(_THREADS)
    assert seen["a_rc"] == -2 and seen["b_rc"] == -1
    assert a_text not in seen["b_before"], seen["b_before"]
    assert seen["b_after"] == [b_text, b_text]
    assert seen["a"] == [a_text, a_text], seen["a"]
