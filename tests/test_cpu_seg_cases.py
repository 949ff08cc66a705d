"""The crafted segmentation cases (tests/seg_cases.py) land where they claim, on the oracle (orc_mfseg_cpu): every threshold quantity is
recomputed here from the inputs (4-connected labelling with scipy, float32 arithmetic in numpy), not taken from the generator, and the
oracle's outputs are checked on the side of each decision.  No GPU."""
from __future__ import annotations

import math

import numpy as np
import pytest
from scipy import ndimage

from tests import seg_cases as sc

f32 = np.float32
CASES = sc.all_cases()
FOUR = np.array([[0, 1, 0], [1, 1, 1], [0, 1, 0]])


def _cc(edges):
    return ndimage.label(edges > 0, structure=FOUR)


def _bijective(a, b):
    """label images equal up to renumbering, 0 <-> 0"""
    if not np.array_equal(a == 0, b == 0):
        return False
    pairs = np.unique(np.stack([a.ravel(), b.ravel()], 1), axis=0)
    return len(set(pairs[:, 0])) == len(pairs) == len(set(pairs[:, 1]))


def _check(case, k, claim, out, cache):
    s = case.steps[k]
    o = out[k]
    kind = claim[0]
    if k not in cache:
        cache[k] = _cc(s.edges)
    lab, n = cache[k]
    P = case.W * case.H
    if kind == "ncomp":
        assert o.nComponents == claim[1] == n + 1
    elif kind == "cc":
        assert o.nComponents == n + 1 and _bijective(o.labels, lab)
    elif kind == "area":
        assert int((lab == lab[claim[1]]).sum()) == claim[2] and lab[claim[1]] > 0
    elif kind == "same":
        assert o.labels[claim[1]] == o.labels[claim[2]] != 0
    elif kind == "diff":
        assert o.labels[claim[1]] != o.labels[claim[2]]
    elif kind == "zero":
        assert o.labels[claim[1]] == 0
    elif kind == "fill":
        _, y, x0, m = claim
        row = o.labels[y]
        assert row[x0 - 1] != 0 and np.all(row[x0:x0 + m] == row[x0 - 1]) and row[x0 + m] == 0
    elif kind == "seg":
        assert o.seg[claim[1]] == claim[2], (o.seg[claim[1]], claim[2])
    elif kind == "new":
        assert (o.hasNew, o.newClass) == (claim[1], claim[2])
    elif kind == "step":
        _, p, q, below = claim
        d0, d1 = f32(s.depth[p]), f32(s.depth[q])
        assert (float(abs(d1 - d0)) < 0.008) == below
        nxt = np.nextafter(d1, f32(np.inf) if (d1 >= d0) == below else f32(-np.inf))      # one ulp towards the other side
        assert (float(abs(nxt - d0)) < 0.008) != below
    elif kind == "t":
        _, p, m, d = claim
        comp = lab == lab[p]
        csize = int(comp.sum())
        t = int(f32(0.65) * f32(csize))
        assert csize > 160 and int((comp & (s.mask == m)).sum()) == t + d
    elif kind == "newsize":
        _, m, which, d = claim
        rel = case.cfg["minRelSizeNew" if which == "min" else "maxRelSizeNew"]
        bound = int(f32(rel) * f32(P))
        assert int((s.mask == m).sum()) == bound + d
        assert all(int((lab == c).sum()) > 160 and np.all(s.mask[lab == c] == m) for c in np.unique(lab[s.mask == m]))   # mask = its components
    elif kind == "ovl":
        _, m, model, d = claim
        mp = int((s.mask == m).sum())
        thr = f32(0.05) * f32(mp)
        ov = int(((s.mask == m) & (s.projected == model)).sum())
        assert ov == math.floor(thr) + d and (ov < thr) == (d < 0)
    elif kind == "absorb":
        _, p, model, d = claim
        csize = int((lab == lab[p]).sum())
        thr = f32(0.6) * f32(csize)
        cnt = int(((o.labels == o.labels[p]) & (s.projected == model)).sum())
        assert cnt == math.floor(thr) + d and (cnt > thr) == (d > 0)
    else:
        raise AssertionError(f"unknown claim {claim}")


@pytest.mark.parametrize("case", CASES, ids=[c.name for c in CASES])
def test_case_lands_where_it_claims(case):
    out = sc.run_oracle(case)
    cache = {}
    assert case.claims
    for k, claim in case.claims:
        try:
            _check(case, k, claim, out, cache)
        except AssertionError as e:
            raise AssertionError(f"{case.name} step {k}: claim {claim} does not hold ({e})") from None


def test_cases_cover_the_issue():
    names = {c.name for c in CASES}
    for (W, H) in sc.CC_SIZES:
        for p in sc.CC_PATTERNS:
            assert f"cc_{p}_{W}x{H}" in names
    assert any(W % 32 and H % 16 for (W, H) in sc.CC_SIZES)              # a remainder tile both ways
    assert any(W <= 32 and H <= 16 for (W, H) in sc.CC_SIZES)            # one tile: no tile edge at all
    assert {"edge_area_49", "edge_area_50", "edge_area_51", "edge_band_8px", "vote_256_masks_63_models"} <= names
    # every pair of neighbour positions two different components can hold (the 8 pairs left out are 4-adjacent)
    pairs = set()
    for c in CASES:
        if c.name.startswith("edge_order_"):
            win = {cl[1]: cl[2] for _, cl in c.claims if cl[0] == "same"}
            for _, cl in c.claims:
                if cl[0] == "diff":
                    (cy, cx), a, b = cl[1], win[cl[1]], cl[2]
                    pairs.add(frozenset([(a[0] - cy, a[1] - cx), (b[0] - cy, b[1] - cx)]))
    assert len(pairs) == 20 and all(abs(p[0] - q[0]) + abs(p[1] - q[1]) > 1 for p, q in map(tuple, pairs))
