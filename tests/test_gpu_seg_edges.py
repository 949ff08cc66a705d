"""The segmentation tail on crafted inputs (tests/seg_cases.py), against the oracle.

Each case runs on a fresh multi-model context through MaskFusion.debugSegment (mf_debug_segment: the kernels of the frame path) and
through orc_mfseg_cpu with one oracle state, call after call, so the ignore map and maskToID carry over on both sides.  fullSegmentation
must match bit for bit, hasNewLabel / newClassID / nComponents exactly, and the labels after edge removal up to a renumbering (one GPU
label per oracle label, 0 <-> 0: the GPU numbers components with an atomic counter).  Run on an H100: pytest -m gpu."""
from __future__ import annotations

import numpy as np
import pytest

from tests import seg_cases as sc

pytestmark = pytest.mark.gpu
CASES = sc.all_cases()


def _context(case):
    import maskfusion_b200 as mfb
    return mfb.MaskFusion(mfb.default_config(case.W, case.H, enableMultipleModels=1, capacityGlobal=20000, **case.cfg))


def _first(bad):
    y, x = np.unravel_index(int(np.argmax(bad)), bad.shape)
    return int(y), int(x)


def _label_mismatch(g, o):
    """None if g and o are the same partition with 0 <-> 0, else the first pixel where the correspondence breaks"""
    if not np.array_equal(g == 0, o == 0):
        return _first((g == 0) != (o == 0))
    og = {}
    go = {}
    gf, of = g.ravel(), o.ravel()
    pairs, first = np.unique(np.stack([gf, of], 1), axis=0, return_index=True)
    for (a, b), i in sorted(zip(map(tuple, pairs), first), key=lambda t: t[1]):
        if og.setdefault(b, a) != a or go.setdefault(a, b) != b:
            return divmod(int(i), g.shape[1])
    return None


@pytest.mark.parametrize("case", CASES, ids=[c.name for c in CASES])
def test_segmentation_matches_oracle(case):
    want = sc.run_oracle(case)
    mf = _context(case)
    try:
        for k, (s, o) in enumerate(zip(case.steps, want)):
            a = case.inputs(s)
            seg, lab, has_new, new_class, n_comp = mf.debugSegment(a["edgesInv"], a["depth"], a["mask"], a["classIDs"], a["projectedIDs"],
                                                                   a["modelIDs"], a["modelClassIDs"], a["nextModelID"], a["allowNew"])
            where = f"{case.name} call {k}"
            assert (has_new, new_class, n_comp) == (o.hasNew, o.newClass, o.nComponents), \
                f"{where}: (hasNewLabel, newClassID, nComponents) cuda {(has_new, new_class, n_comp)} oracle {(o.hasNew, o.newClass, o.nComponents)}"
            bad = _label_mismatch(lab, o.labels)
            assert bad is None, f"{where}: labels after edge removal differ first at (y, x) = {bad}: cuda {lab[bad]} oracle {o.labels[bad]}"
            if not np.array_equal(seg, o.seg):
                p = _first(seg != o.seg)
                raise AssertionError(f"{where}: fullSegmentation differs at {int((seg != o.seg).sum())} pixels, first (y, x) = {p}: "
                                     f"cuda {seg[p]} oracle {o.seg[p]}")
    finally:
        mf.close()


def test_debug_segment_refusals():
    import maskfusion_b200 as mfb
    W, H = 36, 20
    z8, zf = np.zeros((H, W), np.uint8), np.zeros((H, W), np.float32)
    single = mfb.MaskFusion(mfb.default_config(W, H, capacityGlobal=20000))
    try:
        with pytest.raises(mfb.MFError, match="not a multi-model context"):
            single.debugSegment(z8, zf, None, [], z8, [0], [0], 1)
    finally:
        single.close()
    mf = mfb.MaskFusion(mfb.default_config(W, H, enableMultipleModels=1, capacityGlobal=20000))
    try:
        for args in ((z8, list(range(257)), [0], [0], 1), (None, [], [], [], 1), (None, [], list(range(64)), [0] * 64, 1),
                     (None, [], [0], [0], 256), (None, [], [0], [0], -1)):
            mask, cls, ids, mcls, nxt = args
            with pytest.raises(mfb.MFError, match="debug_segment"):
                mf.debugSegment(z8, zf, mask, cls, z8, ids, mcls, nxt)
        with pytest.raises(mfb.MFError, match="no model's"):
            mf.debugSegment(z8, zf, None, [], np.full((H, W), 5, np.uint8), [0], [0], 1)
        with pytest.raises(mfb.MFError, match="below n_masks"):
            mf.debugSegment(z8, zf, np.full((H, W), 2, np.uint8), [0, 1], z8, [0], [0], 1)
        # the largest counts are accepted
        seg, *_ = mf.debugSegment(np.full((H, W), 255, np.uint8), zf, z8, list(range(256)), z8, list(range(63)), [0] * 63, 255)
        assert seg.shape == (H, W)
    finally:
        mf.close()
