"""Convert matterport's Keras Mask R-CNN weights (mask_rcnn_coco.h5) into the safetensors file the library loads.

    python scripts/convert_mrcnn_h5.py mask_rcnn_coco.h5 mask_rcnn_coco.safetensors

then maskfusion_b200.load_mask_rcnn("mask_rcnn_coco.safetensors") (or mf_*_load_weights from C).  Each array keeps its Keras layout and is
stored as float32 under "<layer>/<param>": nested-model prefixes (the RPN lives inside the "rpn_model" sub-model) and the ":0" suffix are
removed, e.g. "rpn_model/rpn_conv_shared/kernel:0" -> "rpn_conv_shared/kernel".  Folding and relayout happen in the library (DESIGN §3c).

The conversion is flatten(), a pure function of {h5 layer: [(weight name, array)]}; read_h5() is the only code that needs h5py.
"""
from __future__ import annotations

import json
import re
import sys

import numpy as np

_DTYPES = {np.dtype(np.float32): "F32", np.dtype(np.float16): "F16", np.dtype(np.float64): "F64", np.dtype(np.int32): "I32"}


def flat_name(layer: str, weight_name: str) -> str:
    """the "<layer>/<param>" name of one Keras weight: the last two path components of its weight name without the ":<n>" suffix (the
    h5 layer's own name where the weight name has a single component)"""
    parts = [p for p in weight_name.split("/") if p]
    param = re.sub(r":\d+$", "", parts[-1])
    return f"{parts[-2] if len(parts) >= 2 else layer}/{param}"


def flatten(layers: dict) -> dict:
    """{h5 layer name: [(weight name, array), ...]} -> {"<layer>/<param>": float32 array}, Keras layouts kept"""
    out = {}
    for layer, weights in layers.items():
        for wname, arr in weights:
            name = flat_name(layer, wname)
            if name in out:
                raise ValueError(f"two weights map to {name!r} (h5 layer {layer!r}, weight {wname!r})")
            out[name] = np.ascontiguousarray(arr, np.float32)
    return out


def write_safetensors(path: str, tensors: dict, metadata: dict | None = None):
    """the safetensors layout: u64 little-endian header length, JSON header (names sorted, padded with spaces to 8 bytes), data"""
    header, blobs, off = {}, [], 0
    for name in sorted(tensors):
        a = np.ascontiguousarray(tensors[name])
        a = a.astype(a.dtype.newbyteorder("<"), copy=False)
        header[name] = {"dtype": _DTYPES[a.dtype.newbyteorder("=")], "shape": list(a.shape), "data_offsets": [off, off + a.nbytes]}
        blobs.append(a.tobytes())
        off += a.nbytes
    if metadata:
        header["__metadata__"] = {str(k): str(v) for k, v in metadata.items()}
    h = json.dumps(header, separators=(",", ":")).encode()
    h += b" " * (-len(h) % 8)
    with open(path, "wb") as f:
        f.write(len(h).to_bytes(8, "little"))
        f.write(h)
        for b in blobs:
            f.write(b)


def read_h5(path: str) -> dict:
    """{h5 layer name: [(weight name, array)]} of a Keras weight file (model.save_weights / the published mask_rcnn_coco.h5)"""
    try:
        import h5py
    except ImportError:
        raise SystemExit("reading .h5 weights needs h5py (pip install h5py); the conversion itself is flatten()")
    layers = {}
    with h5py.File(path, "r") as f:
        g = f["model_weights"] if "model_weights" in f else f
        for layer in g.attrs["layer_names"]:
            layer = layer.decode() if isinstance(layer, bytes) else str(layer)
            names = [n.decode() if isinstance(n, bytes) else str(n) for n in g[layer].attrs["weight_names"]]
            layers[layer] = [(n, np.asarray(g[layer][n])) for n in names]
    return layers


def main(argv):
    if len(argv) != 3:
        raise SystemExit(__doc__)
    tensors = flatten(read_h5(argv[1]))
    write_safetensors(argv[2], tensors, {"source": argv[1].rsplit("/", 1)[-1]})
    print(f"{argv[2]}: {len(tensors)} tensors, {sum(a.size for a in tensors.values())} parameters")


if __name__ == "__main__":
    main(sys.argv)
