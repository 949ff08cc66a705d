"""The crafted surfel cases (tests/surfel_cases.py) hit the edges they claim, checked independently of the generators: numpy float32
projections under the identity pose, the oracle's sprite export against a float64 evaluation of R-PR / R-PC, and the oracle's clean
against the designed survivor count.  No GPU."""
from __future__ import annotations

import ctypes as C
from collections import Counter

import numpy as np
import pytest

from tests import oracle_lib as ol
from tests import surfel_cases as sc
from tests.stagewise import OracleStages

f32 = np.float32


def _proj(store):
    X, Y, Z = store[:, 0], store[:, 1], store[:, 2]
    with np.errstate(divide="ignore", invalid="ignore"):
        return ((sc.FX * X) / Z) + sc.CX, ((sc.FY * Y) / Z) + sc.CY


def _case(name):
    return next(c for c in sc.small_cases() if c.name == name)


@np.errstate(invalid="ignore")
def test_index_edges_claims():
    c = _case("index_edges")
    s = c.store
    x, y = _proj(s)
    Z = s[:, 2]
    ok = (Z > 0) & (Z <= sc.MAXD)
    inner_y = ok & (y > 0) & (y < sc.H) & (y != np.floor(y))
    inner_x = ok & (x > 0) & (x < sc.W) & (x != np.floor(x))
    got = Counter()
    got["x_integer"] = int((inner_y & (x > 0) & (x < sc.W) & (x == np.floor(x))).sum())
    got["x_ulp_below_integer"] = int((inner_y & (x > 1) & (x < sc.W - 1) & (np.floor(x) + 1 - x < 1e-4)).sum())
    got["x_zero"] = int((inner_y & (x == 0)).sum())
    got["x_W_minus_ulp"] = int((inner_y & (x == np.nextafter(f32(sc.W), f32(0)))).sum())
    got["x_W"] = int((inner_y & (x == sc.W)).sum())
    got["y_integer"] = int((inner_x & (y > 0) & (y < sc.H) & (y == np.floor(y))).sum())
    got["y_ulp_below_integer"] = int((inner_x & (y > 1) & (y < sc.H - 1) & (np.floor(y) + 1 - y < 1e-4)).sum())
    got["y_zero"] = int((inner_x & (y == 0)).sum())
    got["y_H_minus_ulp"] = int((inner_x & (y == np.nextafter(f32(sc.H), f32(0)))).sum())
    got["y_H"] = int((inner_x & (y == sc.H)).sum())
    zn = Z / sc.MAXD
    got["z_maxdepth"] = int(((Z == sc.MAXD) & (zn == 1)).sum())
    got["z_maxdepth_minus_ulp"] = int(((Z == np.nextafter(sc.MAXD, f32(0))) & (zn < 1)).sum())
    got["z_maxdepth_plus_ulp"] = int((Z == np.nextafter(sc.MAXD, f32(np.inf))).sum())
    got["z_zero"] = int(((Z == 0) & ~np.signbit(Z)).sum())
    got["z_negzero"] = int(((Z == 0) & np.signbit(Z)).sum())
    # ties: surfels sharing one pixel at bit-identical zn (drawable, inside the image)
    draw = ok & (zn < 1) & (np.floor(x) >= 0) & (np.floor(y) >= 0) & (np.floor(x) < sc.W) & (np.floor(y) < sc.H)
    keys = Counter()
    first = {}
    for i in np.flatnonzero(draw):
        k = (int(np.floor(x[i])), int(np.floor(y[i])), zn[i].view(np.uint32).item())
        keys[k] += 1; first.setdefault(k, i)
    ties = [k for k, n in keys.items() if n >= 2]
    got["tie_groups"] = len(ties)
    got["tie_group_with_id0"] = sum(1 for k in ties if first[k] == 0)
    got["tie_max"] = max(keys[k] for k in ties)
    pix = Counter((int(np.floor(x[i])), int(np.floor(y[i]))) for i in np.flatnonzero(draw))
    stacks = [p for p, n in pix.items() if n >= 100 and len({zn[i].item() for i in np.flatnonzero(draw) if (int(np.floor(x[i])), int(np.floor(y[i]))) == p}) == n]
    got["stack_distinct_depths"] = sum(pix[p] for p in stacks)
    # the lowest-id member of a tie group is not always the first position of the group in x (both id orders)
    orders = set()
    for k in ties:
        ids = [i for i in np.flatnonzero(draw) if (int(np.floor(x[i])), int(np.floor(y[i])), zn[i].view(np.uint32).item()) == k]
        orders.add(bool(x[ids[0]] < x[ids[-1]]))
    assert orders == {True, False}
    for k, v in c.claims.items():
        assert got[k] == v, (k, got[k], v)
    print("index_edges edge classes:", dict(sorted(c.claims.items())))


def test_index_general_claims():
    c = _case("index_general")
    n = c.claims["duplicates"]
    s = c.store
    assert np.array_equal(s[2000:2000 + n].view(np.uint32), s[:n].view(np.uint32))
    assert not np.array_equal(c.pose[:3, :3], np.eye(3, dtype=np.float32))


def _fp32_tie(edge):
    """xw +- s/2 whose float32 rounding lands on a pixel centre although the exact value does not"""
    r = float(f32(edge))
    return r != edge and (r - 0.5) == np.floor(r - 0.5)


def _rule_range(xw, s, W):
    """R-PR (DESIGN section 4): pixels k with xw - s/2 <= k + 0.5 < xw + s/2, in float64 (exact: xw and s are float32, the centres
    half-integers), except that an edge xw +- s/2 whose fp32 rounding lands on a pixel centre is that centre.
    Returns (x0, x1, number of fp32-rounded edges)"""
    e_lo, e_hi = float(xw) - float(s) / 2, float(xw) + float(s) / 2
    t_lo, t_hi = _fp32_tie(e_lo), _fp32_tie(e_hi)
    lo = int(np.ceil((float(f32(e_lo)) if t_lo else e_lo) - 0.5))
    hi = int(np.ceil((float(f32(e_hi)) if t_hi else e_hi) - 0.5)) - 1
    return max(lo, 0), min(hi, W - 1), int(t_lo) + int(t_hi)


SPLAT = [c.name for c in sc.small_cases() if c.kind == "splat"]


@pytest.mark.parametrize("name", SPLAT)
def test_splat_ranges_follow_rule(name):
    """the oracle's R-PC and R-PR decisions for every crafted sprite equal a float64 evaluation of the written rule (DESIGN section 4)"""
    c = _case(name)
    n_ok = n_edge = n_tie = 0
    for s in c.store:
        sp = sc.splat_extent(s, c.pose)
        if not sp.size:
            continue
        inside = 0 <= sp.xw <= sc.W and 0 <= sp.yw <= sc.H
        if not inside:
            assert not sp.ok
            continue
        if not sp.ok:
            continue
        n_ok += 1
        for w, lim, a, b in ((sp.xw, sc.W, sp.x0, sp.x1), (sp.yw, sc.H, sp.y0, sp.y1)):
            lo, hi, ties = _rule_range(w, sp.size, lim)
            e_lo, e_hi = float(w) - float(sp.size) / 2, float(w) + float(sp.size) / 2
            n_edge += int((e_lo - 0.5) == np.floor(e_lo - 0.5)) + int((e_hi - 0.5) == np.floor(e_hi - 0.5))
            n_tie += ties
            assert (a, b) == (lo, hi), (name, float(w), float(sp.size), (a, b), (lo, hi))
    assert n_ok > 0
    if name == "splat_edges":
        assert n_edge >= 32, n_edge          # range endpoints exactly on a pixel centre
        assert n_tie >= 2, n_tie             # edges that only the fp32 rounding puts on a pixel centre, one at each end


def test_splat_edges_claims():
    c = _case("splat_edges")
    got = Counter()
    sps = [sc.splat_extent(s) for s in c.store]
    for s, sp in zip(c.store, sps):
        z = s[2]
        if sp.ok and sp.size == 2047 and sp.x0 == 0 and sp.x1 == sc.W - 1 and sp.y0 == 0 and sp.y1 == sc.H - 1:
            got["size_2047" if s[11] < 30 else "size_above_2047"] += 1
        if sp.ok and 2000 < sp.size < 2047:
            got["size_below_2047"] += 1
        for key, val, lim in (("pc_x", sp.xw, sc.W), ("pc_y", sp.yw, sc.H)):
            if val == 0 and sp.ok:
                got[key + "0"] += 1
            if val == lim and sp.ok:
                got[key + ("W" if key == "pc_x" else "H")] += 1
            if (val < 0 and val > -1e-3) and not sp.ok:
                got[key + "0_outside"] += 1
            if (val > lim and val < lim + 1e-3) and not sp.ok:
                got[key + ("W" if key == "pc_x" else "H") + "_outside"] += 1
        if sp.ok and sp.size < 2046 and float(sp.size).is_integer() and s[11] > 1e-4 and sp.size <= 16 and z == 2.0:
            hits = [((float(w) + sgn * float(sp.size) / 2) - 0.5) % 1 == 0 for w in (sp.xw, sp.yw) for sgn in (-1, 1)]
            got["rpr_exact_size"] += int(all(hits))
        if sp.ok and sp.size == 1 and s[11] <= 1e-5:
            got["size_raw_below_1"] += 1
        if sp.ok:
            e_lo, e_hi = float(sp.xw) - float(sp.size) / 2, float(sp.xw) + float(sp.size) / 2
            # the rounded edge decides: the exact rule would leave pixel x0 out / take pixel x1 + 1 in
            if _fp32_tie(e_lo) and float(f32(e_lo)) < e_lo and sp.x0 + 0.5 < e_lo:
                got["rpr_fp32_tie_lo"] += 1
            if _fp32_tie(e_hi) and float(f32(e_hi)) < e_hi and sp.x1 + 1.5 < e_hi:
                got["rpr_fp32_tie_hi"] += 1
        if z == sc.MAXD:
            got["z_maxdepth"] += int(sp.ok)
        if z == np.nextafter(sc.MAXD, f32(0)):
            got["z_maxdepth_minus_ulp"] += int(sp.ok)
        if z == np.nextafter(sc.MAXD, f32(np.inf)):
            got["z_maxdepth_plus_ulp"] += int(not sp.ok)
        if s[3] == sc.CONF:
            got["conf_eq_threshold"] += int(sp.ok)
        if s[3] == np.nextafter(sc.CONF, f32(0)):
            got["conf_below_threshold"] += int(not sp.ok)
        if s[7] == sc.TICK and abs(s[0] - 0.6) < 1e-6:
            got["last_eq_maxtime"] += int(sp.ok)
        if s[7] == sc.TICK + 1:
            got["last_after_maxtime"] += int(not sp.ok)
    # grazing: |dot(l, n)| of the normal the vertex stage uses and the ray of the pixel the disc was built on
    for i, e in enumerate((1e-1, 1e-3, 1e-5, 1e-7)):
        px, py = 100 + 120 * i, 420
        l = np.array(sc.pixel_ray(px, py), np.float64)
        cands = [sp for s, sp in zip(c.store, sps) if sp.ok and abs(float(s[11]) - 0.02) < 1e-7 and sp.x0 <= px <= sp.x1 and sp.y0 <= py <= sp.y1]
        d = min(abs(float(np.dot(l, sp.n.astype(np.float64)))) for sp in cands)
        got[f"grazing_{e:.0e}"] += int(0.5 * e <= d <= 2 * e if e >= 1e-5 else d < 1e-6)
    # disc rim: the pixel's dot(d, d) against rad^2 (the fragment test of combo_splat.frag in float32)
    for s, sp in zip(c.store, sps):
        if not sp.ok or abs(s[2] - 1.7) > 1e-6:
            continue
        for py in range(sp.y0, sp.y1 + 1):
            for px in range(sp.x0, sp.x1 + 1):
                dd, r2 = sc.disc_dd(sp, px, py)
                if dd == r2:
                    got["rim_eq"] += 1
                elif dd == np.nextafter(r2, f32(np.inf)):
                    got["rim_out"] += 1
                elif dd == np.nextafter(r2, f32(0)):
                    got["rim_in"] += 1
    # coincident surfels, and one-ulp pairs with the nearer one later in the store
    st = c.store
    rows = Counter(r.tobytes() for r in st)
    got["coincident"] = max(n for r, n in rows.items() if np.frombuffer(r, np.float32)[11] < 0.0045)
    got["queue_stack"] = max(rows.values())
    for i in range(1, len(st)):
        a, b = st[i - 1], st[i]
        if a[0] == b[0] and a[1] == b[1] and b[2] == np.nextafter(a[2], f32(0)) and a[2] < 3:
            got["ulp_pair_nearer_later"] += 1
    for k, v in c.claims.items():
        if k.startswith("rim_"):
            assert got[k] >= v, (k, got[k], v)
        else:
            assert got[k] == v, (k, got[k], v)
    q = next(sp for s, sp in zip(c.store, sps) if rows[s.tobytes()] == 48)
    assert (q.x1 - q.x0 + 1) * (q.y1 - q.y0 + 1) * 48 > 64 * 32       # far more than one warp's queue of exact-path fragments
    print("splat_edges edge classes:", dict(sorted(c.claims.items())))


def _oracle_clean(c, conf=None):
    """the oracle's Model::clean after the frame schedule's predictIndices -> fuse -> predictIndices, on the crafted store"""
    cfg = ol.default_config(sc.W, sc.H, **{"capacityGlobal": 1_200_000, **c.cfg})
    st = OracleStages(cfg)
    n = c.store.shape[0]
    m = st.mptr(0).contents
    if n:
        C.memmove(m.surf[m.target], c.store.ctypes.data, c.store.nbytes)
    m.count = n
    for k in range(16):
        m.pose[k] = float(c.pose.ravel()[k]); m.lastPose[k] = float(c.pose.ravel()[k])
    st.set_frame(c.rgb, c.depth); st.tick = sc.TICK
    st.predict_indices(); st.fuse(); st.predict_indices(); st.clean()
    out = st.p.count(0)
    st.p.close()
    return out


CLEAN = [c.name for c in sc.small_cases() if c.kind in ("clean", "time")]


@pytest.mark.parametrize("name", CLEAN)
def test_clean_survivors_as_designed(name):
    c = _case(name)
    assert _oracle_clean(c) == c.survivors, (name, c.survivors)
    if c.removed is not None:
        assert int(c.removed.sum()) == c.claims["removed"]


def test_splat_overshoot_claims():
    """the disc reaches past the sprite at its open upper end: xw + s/2 is exactly the centre of the column after the range, and a pixel
    of that column passes the disc test of combo_splat.frag (so closing the range at an exact centre would draw it)"""
    cases = [c for c in sc.small_cases() if "rpr_hi_edge_in_disc" in c.claims]
    assert len(cases) >= 2
    for c in cases:
        (s,) = c.store
        sp = sc.splat_extent(s, c.pose)
        col = sp.x1 + 1
        assert sp.ok and col < sc.W and float(sp.xw) + float(sp.size) / 2 == col + 0.5
        inside = [py for py in range(sp.y0, sp.y1 + 1) if np.less_equal(*sc.disc_dd(sp, col, py))]
        assert inside, c.name
        fd = (sp.pos[2] / (2 * sc.MAXD)) + 0.5
        assert fd < 1


def test_clean_big_survivors_as_designed():
    plane, zero = sc.big_cases()
    assert plane.claims["clamped"] == 1 and plane.claims["frame"] == "plane" and plane.store.shape[0] > 1_000_000
    assert _oracle_clean(plane) == plane.survivors == plane.cfg["capacityGlobal"]
    assert zero.claims["frame"] == "zero" and zero.store.shape[0] == plane.store.shape[0] and zero.claims["removed"] == 1
    assert _oracle_clean(zero) == zero.survivors == zero.store.shape[0] - 1


def test_clean_claims():
    cases = {c.name: c for c in sc.small_cases()}
    a = cases["clean_attrs"]
    s = a.store
    x, y = _proj(s)
    vis = (s[:, 2] > 0) & (x > 0) & (y > 0) & (x < sc.W) & (y < sc.H)
    assert int(vis.sum()) == a.claims["visible"] and int((s[:, 2] < 0).sum()) == a.claims["behind_camera"]
    lt, cf = s[:, 7], s[:, 3]
    below = np.nextafter(sc.CONF, f32(0))
    got = {"last_minus1": int((lt == -1).sum()), "last_minus2": int(((lt == -2) & (cf > sc.CONF)).sum()),
           "last_minus2_lowconf": int(((lt == -2) & (cf == below)).sum()),
           "age20_conf_below": int(((sc.TICK - lt == 20) & (cf == below)).sum()), "age20_conf_eq": int(((sc.TICK - lt == 20) & (cf == sc.CONF)).sum()),
           "age21_conf_eq": int(((sc.TICK - lt == 21) & (cf == sc.CONF)).sum()), "age21_conf_below": int(((sc.TICK - lt == 21) & (cf == below)).sum()),
           "age21_conf_above": int(((sc.TICK - lt == 21) & (cf > sc.CONF)).sum())}
    for k, v in got.items():
        assert a.claims[k] == v, (k, v)
    pats = Counter()
    for c in cases.values():
        if c.kind != "clean" or c.removed is None:
            continue
        pats[c.claims["pattern"]] += 1
        n, r = c.store.shape[0], c.removed
        if c.claims["pattern"] == "511_512_513" and n > 513:
            assert r[511] and r[512] and r[513] and r.sum() == 3
        if c.claims["pattern"] == "runs":
            assert r[300:420].all() and r[2047:2049].all()
    counts = Counter(c.store.shape[0] for c in cases.values() if c.kind == "clean")
    for n in (0, 1, 511, 512, 513):
        assert counts[n] == 2, n
    assert sum(c.claims.get("clamped", 0) for c in cases.values()) >= 2 and sum(c.claims.get("full", 0) for c in cases.values()) >= 2
    print("clean patterns:", dict(sorted(pats.items())), "store counts:", dict(sorted(counts.items())))


def test_time_gate_claims():
    c = _case("time_gates")
    dt = sc.TICK - c.store[:, 7]
    assert int((dt == sc.TIME_DELTA).sum()) == c.claims["dt_eq"] and int((dt == sc.TIME_DELTA + 1).sum()) == c.claims["dt_above"]
    # drawn into the index map (gate `time - last > delta` false at equality) but outside clean's strict window gate: the fused noWindow path
    x, y = _proj(c.store)
    vis = (c.store[:, 2] > 0) & (x > 0) & (y > 0)
    assert int((vis & (dt == sc.TIME_DELTA)).sum()) >= 1
    old = (dt > 20) & (c.store[:, 3] < sc.CONF)
    assert int(old.sum()) == c.claims["dt_old_lowconf"]          # removed by age, kept again by the time gate


def test_case_inventory(capsys):
    """every edge class of the three passes has a case; prints the number of cases per class (also under -q)"""
    per = Counter()
    for c in sc.all_cases():
        for k, v in c.claims.items():
            if isinstance(v, int) and v and k not in ("count", "removed", "visible", "tail"):
                per[f"{c.kind}:{k}"] += 1
        per[f"{c.kind}:cases"] += 1
    with capsys.disabled():
        print("\ncases per edge class:", ", ".join(f"{k} {v}" for k, v in sorted(per.items())))
    for k in ("index:x_zero", "index:x_W", "index:tie_group_with_id0", "index:z_maxdepth", "index:z_negzero", "clean:clamped", "clean:full",
              "clean:last_minus1", "clean:age21_conf_eq", "splat:pc_xW", "splat:rpr_exact_size", "splat:size_2047", "splat:grazing_1e-07",
              "splat:rim_eq", "splat:queue_stack", "splat:rpr_hi_edge_in_disc", "splat:rpr_fp32_tie_lo", "splat:rpr_fp32_tie_hi",
              "time:dt_eq"):
        assert per[k] >= 1, k
