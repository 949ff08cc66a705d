"""Pretrained Mask R-CNN weights on the host (csrc/mf_weights.cu through mf_mrcnn_read_layer, no CUDA device): the safetensors reader,
R-FOLD and the relayout into the handles' tables bit for bit against the numpy restatement (tests/mrcnn_weights_ref.py), the refusals of
corrupted files, and the h5 converter's name flattening (scripts/convert_mrcnn_h5.py)."""
from __future__ import annotations

import importlib.util
import json
import os
import zlib

import numpy as np
import pytest

from tests import mrcnn_weights_ref as ref

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _converter():
    spec = importlib.util.spec_from_file_location("convert_mrcnn_h5", os.path.join(ROOT, "scripts", "convert_mrcnn_h5.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


conv = _converter()


def _layer_tensors(handle_layer: str, seed: int) -> dict:
    """the Keras arrays of one handle layer (kernel, bias and BatchNorm of each part), drawn like ref.make_weights"""
    parts = {n: p for tabs in ref.handle_tables().values() for n, p, _, _ in tabs}[handle_layer]
    rng = np.random.default_rng(seed)
    shapes = {n: s for layers in ref.ALL_LAYERS.values() for n, _, s in layers}
    bns = {n: bn for layers in ref.ALL_LAYERS.values() for n, bn, _ in layers}
    t = {}
    for name in parts:
        s = shapes[name]
        cout = s[2] if name == "mrcnn_mask_deconv" else s[-1]
        t[f"{name}/kernel"] = (rng.standard_normal(s) * 0.05).astype(np.float32)
        t[f"{name}/bias"] = rng.standard_normal(cout).astype(np.float32)
        if bns[name]:
            bn = bns[name]
            t[f"{bn}/gamma"] = rng.uniform(0.1, 2.0, cout).astype(np.float32)
            t[f"{bn}/beta"] = rng.standard_normal(cout).astype(np.float32)
            t[f"{bn}/moving_mean"] = rng.standard_normal(cout).astype(np.float32)
            t[f"{bn}/moving_variance"] = rng.uniform(1e-4, 3.0, cout).astype(np.float32)      # near 0: eps matters
    return t


KINDS = ["conv1",                                  # stem conv + BN, K 147 padded to 192
         "res3a_branch2b",                         # 3x3 conv + BN
         "res4w_branch2c",                         # the last identity block of stage 4
         "fpn_c3p3",                               # conv + bias (FPN)
         "rpn_class_raw+rpn_bbox_pred",            # RPN head pair, 18 rows padded to 64
         "mrcnn_class_conv1",                      # FC1: 7x7 conv + BN
         "mrcnn_class_logits+mrcnn_bbox_fc",       # dense pair, 405 rows padded to 448
         "mrcnn_mask_conv2",                       # mask conv + BN
         "mrcnn_mask_deconv",                      # transposed conv
         "mrcnn_mask"]                             # mask logits, 81 rows padded to 128


@pytest.mark.parametrize("layer", KINDS)
def test_read_layer_matches_numpy_fold(product_lib, tmp_path, layer):
    t = _layer_tensors(layer, zlib.crc32(layer.encode()))
    extra = {"rpn_model/other/kernel": np.ones((3, 3), np.float16), "unused/kernel": np.zeros(5, np.float32)}     # ignored (by_name)
    path = str(tmp_path / "w.safetensors")
    conv.write_safetensors(path, {**t, **extra}, {"format": "np"})
    w, b = product_lib.read_mrcnn_layer(path, layer)
    W, B = ref.table(t, layer)
    assert w.shape == W.shape and b.shape == B.shape
    assert np.array_equal(w.view(np.uint32), W.view(np.uint32)), np.argwhere(w.view(np.uint32) != W.view(np.uint32))[:5]
    assert np.array_equal(b.view(np.uint32), B.view(np.uint32))
    used = sum(t[k].shape[-1] if k.endswith("/kernel") and "deconv" not in k else 0 for k in t)
    rows = 1024 if layer == "mrcnn_mask_deconv" else used
    assert not w[rows:].any() and not b[rows:].any()                                  # padding rows
    k = t[layer.split("+")[0] + "/kernel"]
    cols = k.shape[3] if layer == "mrcnn_mask_deconv" else k[..., 0].size
    assert not w[:, cols:].any()                                                      # padding columns
    assert (w[:rows, :cols] != 0).mean() > 0.99


def test_name_table_matches_the_library(product_lib):
    """every handle layer of the numpy table exists in the library with the same [rows x K]; unknown names are refused"""
    import ctypes as C
    L = product_lib.load_library()
    n = 0
    for part, tabs in ref.handle_tables().items():
        for name, _, rows, K in tabs:
            d = np.zeros(2, np.int32)
            assert L.mf_mrcnn_read_layer(b"/nonexistent", name.encode(), None, None, d.ctypes.data_as(C.c_void_p)) == 0, name
            assert d.tolist() == [rows, K], (name, d.tolist())
            n += 1
    assert n == 112 + 2 + 9
    assert len(ref.make_weights(0, ("rpn",))) == 6
    with pytest.raises(product_lib.MFError, match="no layer named 'res4x_branch2a'"):
        product_lib.read_mrcnn_layer("/nonexistent", "res4x_branch2a")


def test_reads_files_written_by_safetensors(product_lib, tmp_path):
    st = pytest.importorskip("safetensors.numpy")
    t = _layer_tensors("mrcnn_mask_conv4", 4)
    a, b = str(tmp_path / "lib.safetensors"), str(tmp_path / "ours.safetensors")
    st.save_file(t, a)
    conv.write_safetensors(b, t)
    for p in (a, b):
        w, bias = product_lib.read_mrcnn_layer(p, "mrcnn_mask_conv4")
        W, B = ref.table(t, "mrcnn_mask_conv4")
        assert np.array_equal(w.view(np.uint32), W.view(np.uint32)) and np.array_equal(bias.view(np.uint32), B.view(np.uint32))
    back = st.load_file(b)
    assert set(back) == set(t) and all(np.array_equal(back[k], t[k]) for k in t)


# ---- refusals ---------------------------------------------------------------------------------------------------------------------
LAYER = "fpn_c2p2"


def _raw(header, data: bytes, hlen=None) -> bytes:
    h = header if isinstance(header, bytes) else json.dumps(header).encode()
    return (len(h) if hlen is None else hlen).to_bytes(8, "little") + h + data


def _good():
    t = _layer_tensors(LAYER, 9)
    header, off, data = {}, 0, b""
    for k in sorted(t):
        header[k] = {"dtype": "F32", "shape": list(t[k].shape), "data_offsets": [off, off + t[k].nbytes]}
        data += t[k].tobytes(); off += t[k].nbytes
    return header, data


def _refused(product_lib, tmp_path, blob: bytes, *must):
    p = str(tmp_path / "bad.safetensors")
    with open(p, "wb") as f:
        f.write(blob)
    with pytest.raises(product_lib.MFError) as e:
        product_lib.read_mrcnn_layer(p, LAYER)
    msg = str(e.value)
    assert p in msg, msg
    for m in must:
        assert m in msg, (m, msg)
    return msg


def _edit(header, name, **kw):
    h = json.loads(json.dumps(header))
    h[name].update(kw)
    return h


def test_refusals_name_the_file_and_tensor(product_lib, tmp_path):
    header, data = _good()
    K, Bn = f"{LAYER}/kernel", f"{LAYER}/bias"
    p = str(tmp_path / "ok.safetensors")
    with open(p, "wb") as f:
        f.write(_raw(header, data))
    product_lib.read_mrcnn_layer(p, LAYER)                                            # the unedited file loads
    # truncated data / header length beyond the file
    _refused(product_lib, tmp_path, _raw(header, data[:-4]), "data_offsets", "truncated")
    _refused(product_lib, tmp_path, _raw(header, data, hlen=len(json.dumps(header)) + len(data) + 1), "larger than the file")
    _refused(product_lib, tmp_path, b"\x10\x00\x00", "truncated")
    # JSON outside the grammar
    for bad in (b'{"a":{"dtype":"F32","shape":[1],"data_offsets":[0,4]},}', b'{"a":{"dtype":"F32","shape":[1.5],"data_offsets":[0,4]}}',
                b'{"a":{"dtype":"F32","shape":[-1],"data_offsets":[0,4]}}', b'{"a":{"dtype":"F32","shape":[1]}}',
                b'{"a":{"dtype":"F32","shape":[1],"data_offsets":[0,4],"x":1}}', b'{"a":{"dtype":"F32","shape":[1],"data_offsets":[0,4,8]}}',
                b'{"a":{"dtype":"F32","shape":[01],"data_offsets":[0,4]}}', b'["a"]', b'{"a":{"dtype":F32}}'):
        _refused(product_lib, tmp_path, _raw(bad, b"\0" * 8), "bad header JSON", "'a'" if bad[:2] == b'{"' else "")
    _refused(product_lib, tmp_path, _raw(json.dumps(header).encode() + b"}", data), "trailing bytes")
    dup = json.dumps(header).encode()[:-1] + b',"%s":' % K.encode() + json.dumps(header[K]).encode() + b"}"
    _refused(product_lib, tmp_path, _raw(dup, data), K, "repeated name")
    # dtype, shape, offsets, missing
    _refused(product_lib, tmp_path, _raw(_edit(header, K, dtype="F16"), data), K, "F16")
    _refused(product_lib, tmp_path, _raw(_edit(header, K, shape=[1, 1, 256, 128]), data), K, "(1, 1, 256, 128)", "(1, 1, 256, 256)")
    _refused(product_lib, tmp_path, _raw(_edit(header, Bn, shape=[256, 1]), data), Bn, "shape")
    o = header[K]["data_offsets"]
    _refused(product_lib, tmp_path, _raw(_edit(header, K, data_offsets=[o[0], len(data) + 4]), data), K, "outside")
    _refused(product_lib, tmp_path, _raw(_edit(header, K, data_offsets=[o[1], o[0]]), data), K, "outside")
    _refused(product_lib, tmp_path, _raw(_edit(header, K, data_offsets=[o[0], o[1] - 4]), data), K, "bytes")
    h = json.loads(json.dumps(header)); del h[Bn]
    _refused(product_lib, tmp_path, _raw(h, data), Bn, "missing")


def test_corrupted_file_sweep(product_lib, tmp_path):
    """random byte edits, truncations and header-length changes of a valid file: every result is a clean refusal or a clean load (an edit
    inside the data section), never a crash"""
    header, data = _good()
    good = _raw(header, data)
    hl = int.from_bytes(good[:8], "little")
    rng = np.random.default_rng(17)
    p = str(tmp_path / "fuzz.safetensors")
    refused = loaded = 0
    cases = [good[:n] for n in list(range(0, 8 + hl + 9)) + rng.integers(8 + hl, len(good), 40).tolist()]
    for _ in range(600):
        b = bytearray(good)
        for pos in rng.integers(0, 8 + hl, rng.integers(1, 4)):
            b[pos] = int(rng.choice([rng.integers(0, 256), ord(rng.choice(list('{}[]",:0123456789 ')))]))
        cases.append(bytes(b))
    cases += [(hl + d).to_bytes(8, "little") + good[8:] for d in (-hl, -1, 1, 7, len(data), 1 << 40)]
    for blob in cases:
        with open(p, "wb") as f:
            f.write(blob)
        try:
            product_lib.read_mrcnn_layer(p, LAYER)
            loaded += 1
        except product_lib.MFError as e:
            assert p in str(e)
            refused += 1
    assert refused > 400 and loaded >= 1, (refused, loaded)


# ---- converter ----------------------------------------------------------------------------------------------------------------------
def test_converter_flattens_nested_keras_names():
    a = lambda *s: np.arange(int(np.prod(s)), dtype=np.float64).reshape(s)
    layers = {
        "conv1": [("conv1/kernel:0", a(7, 7, 3, 64)), ("conv1/bias:0", a(64))],
        "bn_conv1": [("bn_conv1/gamma:0", a(64)), ("bn_conv1/beta:0", a(64)), ("bn_conv1/moving_mean:0", a(64)),
                     ("bn_conv1/moving_variance:0", a(64))],
        "rpn_model": [("rpn_conv_shared/kernel:0", a(3, 3, 256, 512)), ("rpn_conv_shared/bias:0", a(512)),
                      ("rpn_model/rpn_class_raw/kernel:0", a(1, 1, 512, 6)), ("rpn_model/rpn_class_raw/bias:0", a(6))],
        "mrcnn_class_conv1": [("mrcnn_class_conv1/kernel:0", a(7, 7, 256, 1024))],
        "mrcnn_mask_deconv": [("kernel:0", a(2, 2, 256, 256))],
        "input_image": [],
    }
    out = conv.flatten(layers)
    assert sorted(out) == sorted(["conv1/kernel", "conv1/bias", "bn_conv1/gamma", "bn_conv1/beta", "bn_conv1/moving_mean",
                                  "bn_conv1/moving_variance", "rpn_conv_shared/kernel", "rpn_conv_shared/bias", "rpn_class_raw/kernel",
                                  "rpn_class_raw/bias", "mrcnn_class_conv1/kernel", "mrcnn_mask_deconv/kernel"])
    assert all(v.dtype == np.float32 for v in out.values())
    assert out["rpn_class_raw/kernel"].shape == (1, 1, 512, 6) and np.array_equal(out["conv1/bias"], np.arange(64, dtype=np.float32))
    with pytest.raises(ValueError, match="rpn_conv_shared/kernel"):
        conv.flatten({"rpn_model": [("rpn_conv_shared/kernel:0", a(1))], "x": [("rpn_model/rpn_conv_shared/kernel:0", a(1))]})


def test_converter_output_loads(product_lib, tmp_path):
    """the converter's file of nested Keras names carries the layer the library reads"""
    t = _layer_tensors("rpn_class_raw+rpn_bbox_pred", 2)
    layers = {"rpn_model": [(f"rpn_model/{k}:0", v.astype(np.float64)) for k, v in t.items()]}
    path = str(tmp_path / "c.safetensors")
    conv.write_safetensors(path, conv.flatten(layers), {"source": "test"})
    w, b = product_lib.read_mrcnn_layer(path, "rpn_class_raw+rpn_bbox_pred")
    W, B = ref.table(t, "rpn_class_raw+rpn_bbox_pred")
    assert np.array_equal(w, W) and np.array_equal(b, B)
