"""Ownership of CUDA resources in the library sources: device memory, pinned host memory, events and streams are acquired and released only
by the owner types next to DevBuf in mf_kernels.h (DevBuf, HostBuf, Event, Stream).  Everything else holds an owner, so a throw in a
constructor releases what it had acquired, and no destructor frees a handle by hand."""
from __future__ import annotations

import os
import re

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "maskfusion_b200", "csrc")
OWNERS = ("DevBuf", "HostBuf", "Event", "Stream")
CALL = re.compile(r"\b(cudaMalloc\w*|cudaFree\w*|cudaHostAlloc|cudaEventCreate\w*|cudaEventDestroy|cudaStreamCreate\w*|cudaStreamDestroy)\s*\(")


def _owner_spans(text: str):
    """[start, end) of the body of every owner type defined in text"""
    spans = []
    for name in OWNERS:
        m = re.search(r"\bstruct\s+%s\s*\{" % name, text)
        if not m:
            continue
        depth = 0
        for i in range(m.end() - 1, len(text)):
            depth += {"{": 1, "}": -1}.get(text[i], 0)
            if depth == 0:
                spans.append((m.start(), i + 1))
                break
    return spans


def test_resource_calls_only_inside_the_owner_types():
    stray = []
    for f in sorted(os.listdir(CSRC)):
        text = open(os.path.join(CSRC, f)).read()
        spans = _owner_spans(text) if f == "mf_kernels.h" else []
        for m in CALL.finditer(text):
            if not any(a <= m.start() < b for a, b in spans):
                stray.append(f"{f}:{text.count(chr(10), 0, m.start()) + 1}: {m.group(1)}")
    assert not stray, "CUDA resources acquired or released outside the owner types:\n" + "\n".join(stray)
    assert len(_owner_spans(open(os.path.join(CSRC, "mf_kernels.h")).read())) == len(OWNERS)
