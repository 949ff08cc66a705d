"""In-tree build of the CUDA library (sm_90a only).

    python -m maskfusion_b200.build [--force]

nvcc cross-compiles without a GPU.  The resulting libmaskfusion_b200.so sits next to this
file (git-ignored).  Flags:
  -gencode arch=compute_90a,code=sm_90a     Hopper H100 only, no fallback architectures
                                            (wgmma, TMA and clusters need the "a" target)
  -fmad=false                               per-element kernels must reproduce IEEE fp32
                                            results bit for bit (parity contract, DESIGN.md)
  -lineinfo                                 ncu source pages map to these files
"""
from __future__ import annotations

import os
import subprocess
import sys
from concurrent.futures import ThreadPoolExecutor

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
# A/B experiments: MFB200_DEFINES="-DPT_THREADS=544 ..." MFB200_TAG=alt builds libmaskfusion_b200_alt.so next to the default library
TAG = os.environ.get("MFB200_TAG", "")
EXTRA_DEFINES = os.environ.get("MFB200_DEFINES", "").split()
OUT = os.path.join(HERE, "libmaskfusion_b200%s.so" % ("_" + TAG if TAG else ""))
OBJ_DIR = os.path.join(HERE, "build" + ("_" + TAG if TAG else ""))
NVCC = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")

ARCH = ["-gencode", "arch=compute_90a,code=sm_90a"]
COMMON = ["-O3", "-std=c++17", "-lineinfo", "-Xcompiler", "-fPIC", "--expt-relaxed-constexpr"]
# file -> extra flags
SOURCES = {
    "mf_frame.cu": ["-fmad=false"],
    "mf_surfel.cu": ["-fmad=false"],
    "mf_seg.cu": ["-fmad=false"],
    "mf_track.cu": ["-fmad=false"],
    "mf_host.cu": ["-fmad=false"],
    "mf_sched.cu": ["-fmad=false"],       # device-side lifecycle of the multi-model schedule + the NCCL exchange (libnccl via dlopen)
    "mf_capi.cu": ["-fmad=false"],
    "mf_jpeg.cu": [],                     # host code only: baseline JPEG decode, libjpeg's default path restated
    "mf_loader.cu": [],                   # host code only: image-directory loader (PNG/PNM decode, zlib)
    "mf_cnn.cu": [],                      # tensor-core GEMMs: no bit-exactness contract, FMA contraction on
    "mf_rpn.cu": ["-fmad=false"],         # proposal layer + ROI Align: bit-exact against the numpy restatement (the GEMMs live in mf_cnn.cu)
    "mf_heads.cu": ["-fmad=false"],       # detection layer, mask select, unmould + id image: bit-exact against the numpy restatement
    "mf_weights.cu": ["-Xcompiler", "-ffp-contract=off"],   # host code only: safetensors weights, R-FOLD bit-exact against numpy
}


def _deps():
    return [os.path.join(CSRC, f) for f in os.listdir(CSRC)] + [os.path.join(HERE, "..", "include", "maskfusion_b200.h"), __file__]


def needs_build() -> bool:
    if not os.path.exists(OUT):
        return True
    t = os.path.getmtime(OUT)
    return any(os.path.getmtime(d) > t for d in _deps())


def _compile(src: str, verbose: bool):
    obj = os.path.join(OBJ_DIR, src.replace(".cu", ".o"))
    srcp = os.path.join(CSRC, src)
    hdrs = [os.path.join(CSRC, f) for f in os.listdir(CSRC) if f.endswith((".h", ".cuh"))]
    hdrs.append(os.path.join(HERE, "..", "include", "maskfusion_b200.h"))
    if os.path.exists(obj) and all(os.path.getmtime(obj) > os.path.getmtime(d) for d in [srcp, __file__] + hdrs):
        return obj
    cmd = [NVCC] + ARCH + COMMON + SOURCES[src] + EXTRA_DEFINES + ["-c", srcp, "-o", obj]
    if verbose:
        cmd += ["-Xptxas", "-v"]
    r = subprocess.run(cmd, capture_output=True, text=True)
    if r.returncode != 0:
        raise RuntimeError(f"nvcc failed for {src}:\n{r.stdout}\n{r.stderr}")
    if verbose:
        sys.stderr.write(r.stderr)
    return obj


def build(force: bool = False, verbose: bool = False) -> str:
    if not force and not needs_build():
        return OUT
    os.makedirs(OBJ_DIR, exist_ok=True)
    if force:
        for f in os.listdir(OBJ_DIR):
            os.remove(os.path.join(OBJ_DIR, f))
    with ThreadPoolExecutor(max_workers=6) as ex:
        objs = list(ex.map(lambda s: _compile(s, verbose), SOURCES))
    cmd = [NVCC] + ARCH + ["-shared", "-o", OUT] + objs + ["-lz", "-lcudart", "-ldl"]
    r = subprocess.run(cmd, capture_output=True, text=True)
    if r.returncode != 0:
        raise RuntimeError(f"link failed:\n{r.stdout}\n{r.stderr}")
    return OUT


if __name__ == "__main__":
    print(build(force="--force" in sys.argv, verbose="-v" in sys.argv))
