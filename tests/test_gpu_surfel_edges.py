"""The surfel passes on crafted stores (tests/surfel_cases.py), bit for bit against the oracle.

Each case is loaded into a fresh context (uploadMap + debugSetPoses) and into OracleStages (the store copied into the model, pose and
last pose set), then run through the frame schedule's stages: combinedPredict on the store as given, then setFrame -> predictIndices ->
fuse -> predictIndices -> clean -> combinedPredict.  After each stage every output is compared as bit patterns.  The variants of
Model::clean (index map fused into pass 1, flushed before it, window read from the three images; in-place and ping-pong compaction)
and both grid shapes of the splat rasteriser are run explicitly, and the kernels that ran are asserted where their names show it.
Run on an H100: pytest -m gpu."""
from __future__ import annotations

import ctypes as C

import numpy as np
import pytest

from tests import oracle_lib as ol
from tests import surfel_cases as sc
from tests.stagewise import OracleStages
from tests.test_gpu_parity import Report

pytestmark = pytest.mark.gpu

SMALL_CAP = 400_000          # < 2^20: splat grid of (columns, 8) blocks; in-place compaction
LARGE_CAP = 1 << 20          # >= 2^20: persistent splat grid; ping-pong compaction after a clean that moved > 40 % of the store


class BitReport(Report):
    def bits(self, what, a, b):
        a = np.ascontiguousarray(a); b = np.ascontiguousarray(b)
        if a.shape != b.shape:
            self.check(what, False, f"shapes {a.shape} vs {b.shape}")
            return
        if a.dtype.kind == "f":
            ua, ub = a.view(np.uint32 if a.itemsize == 4 else np.uint64), b.view(np.uint32 if b.itemsize == 4 else np.uint64)
            bad = (ua != ub) & ~(np.isnan(a) & np.isnan(b))
        else:
            bad = a != b
        n = int(bad.sum())
        first = np.unravel_index(int(np.argmax(bad)), bad.shape) if n else None
        self.check(what, n == 0, f"mismatches={n}/{a.size}" + (f" first at {tuple(int(i) for i in first)}: {a[first]!r} vs {b[first]!r}" if n else ""))


def _load(case, gm, orc):
    n = case.store.shape[0]
    gm.uploadMap(case.store if n else np.zeros((0, 12), np.float32))
    gm.debugSetPoses(case.pose, case.pose)
    m = orc.mptr(0).contents
    if n:
        C.memmove(m.surf[m.target], case.store.ctypes.data, case.store.nbytes)
    m.count = n
    for k in range(16):
        m.pose[k] = float(case.pose.ravel()[k]); m.lastPose[k] = float(case.pose.ravel()[k])


def _prime_ping_pong(gm, mf, case):
    """one clean of a one-surfel store: its removal moves every sub-block, so the next clean of this context copies (ping-pong)"""
    gm.uploadMap(sc.surfel(0.0, 0.0, -1.0, last=-1)[None, :])
    gm.debugSetPoses(case.pose, case.pose)
    mf.setFrame(case.rgb, case.depth)
    gm.predictIndices(sc.TICK); gm.clean(sc.TICK)
    mf.sync()                                    # the statistic that selects the copy is read back without waiting


def _splat(rep, tag, gm, orc):
    orc.predict(); gm.combinedPredict(sc.TICK, sc.TICK)
    im, vc, nr, tt = gm.prediction()
    rep.bits(f"{tag} splat image", im, orc.p.tex(0, "splatImage"))
    rep.bits(f"{tag} splat vertex", vc, orc.p.tex(0, "splatVertex"))
    rep.bits(f"{tag} splat normal", nr, orc.p.tex(0, "splatNormal"))
    rep.bits(f"{tag} splat time", tt, orc.p.tex(0, "splatTime"))
    fim, fv, fn = gm.fillIn()
    rep.bits(f"{tag} fill image", fim, orc.p.tex(0, "fillImage"))
    rep.bits(f"{tag} fill vertex", fv, orc.p.tex(0, "fillVertex"))
    rep.bits(f"{tag} fill normal", fn, orc.p.tex(0, "fillNormal"))
    return int((orc.p.tex(0, "splatImage")[..., 3] > 0).sum())


def _index(rep, tag, gm, orc):
    idx, vc, ct, nr = gm.indexMap()
    rep.bits(f"{tag} index ids", idx, orc.p.tex(0, "idx"))
    rep.bits(f"{tag} index vertConf", vc, orc.p.tex(0, "vertConf"))
    rep.bits(f"{tag} index colorTime", ct, orc.p.tex(0, "colorTime"))
    rep.bits(f"{tag} index normRad", nr, orc.p.tex(0, "normRad"))


def run_case(case, cap, window="fused", ping_pong=False):
    import maskfusion_b200 as mfb
    kw = {**case.cfg, "capacityGlobal": cap}
    rep = BitReport(f"surfel_{case.name}_{cap}_{window}_{'pingpong' if ping_pong else 'inplace'}")
    orc = OracleStages(ol.default_config(sc.W, sc.H, **kw))
    mf = mfb.MaskFusion(mfb.default_config(sc.W, sc.H, **kw))
    try:
        gm = mf.getBackgroundModel()
        if ping_pong:
            _prime_ping_pong(gm, mf, case)
        _load(case, gm, orc)
        orc.set_frame(case.rgb, case.depth); mf.setFrame(case.rgb, case.depth)
        orc.tick = sc.TICK
        drawn = _splat(rep, "[given]", gm, orc)
        orc.predict_indices(); gm.predictIndices(sc.TICK)
        _index(rep, "[index 1]", gm, orc)
        orc.fuse(); gm.fuse(sc.TICK, mf.cfg.depthCutoff, 1.0)
        flag, best, meas = gm.association()
        fo, bo, mo = orc.p.tex(0, "updateId"), orc.p.tex(0, "best"), orc.p.tex(0, "meas")
        rep.bits("[fuse] assoc flags", flag, fo)
        rep.bits("[fuse] assoc best", best[fo == 1], bo[fo == 1])
        rep.bits("[fuse] assoc meas", meas[fo > 0], mo[fo > 0])
        rep.bits("[fuse] store", gm.downloadMap(), orc.p.surfels(0))
        orc.predict_indices(); gm.predictIndices(sc.TICK)
        if window != "fused":
            _index(rep, "[index 2, flushed]", gm, orc)
        if window == "images":
            # the packed window texels were resolved with the old threshold: Model::clean reads the three index-map images
            conf = float(np.nextafter(sc.CONF, np.float32(np.inf)))
            orc.mptr(0).contents.confThreshold = conf; gm.setConfidenceThreshold(conf)
        mf.setProfiling(True)
        orc.clean(); gm.clean(sc.TICK)
        ran = mf.stageTimes()
        mf.setProfiling(False)
        # What the kernel names can show: whether the index projection ran inside clean (fused) or before it, and which compaction ran.
        # The packed and the image window are two instantiations of one kernel name (k_clean_p2), so the images variant is asserted only
        # as "not fused" with a threshold that differs from the one the index map was resolved with; likewise both splat grid shapes
        # launch k_splat_project, and the shape follows from the capacity alone (splatGrid: persistent at >= 2^20, else 8 rows).
        if window == "fused":
            rep.check("index projection fused into clean pass 1", "k_index_project" not in ran and "k_index_resolve" in ran, str(sorted(ran)))
            _index(rep, "[index 2, fused, read after clean]", gm, orc)
        else:
            rep.check("index map resolved before clean", "k_index_resolve" not in ran and "k_index_project" not in ran, str(sorted(ran)))
        rep.check("compaction", ("k_clean_scatter" if ping_pong else "k_clean_compact") in ran
                  and ("k_clean_compact" if ping_pong else "k_clean_scatter") not in ran, str(sorted(ran)))
        so, sm = orc.p.surfels(0), gm.downloadMap()
        rep.check("[clean] count", so.shape[0] == sm.shape[0], f"{so.shape[0]} vs {sm.shape[0]}")
        if case.survivors is not None:
            rep.check("[clean] designed count", so.shape[0] == case.survivors, f"{so.shape[0]} vs {case.survivors}")
        rep.bits("[clean] store (ordered)", sm, so)
        _splat(rep, "[predict]", gm, orc)
        rep.log.append(f"pixels drawn from the crafted store: {drawn}")
    finally:
        mf.close(); orc.p.close()
    rep.finish()
    return drawn


def _runs():
    runs = []
    for c in sc.small_cases():
        if c.kind == "index":
            runs += [(c.name, SMALL_CAP, w, False) for w in ("fused", "flushed", "images")]
        elif c.kind == "time":
            runs += [(c.name, SMALL_CAP, w, False) for w in ("fused", "flushed")]
        elif c.kind == "splat":
            runs += [(c.name, SMALL_CAP, "fused", False), (c.name, LARGE_CAP, "fused", False)]
        else:
            cap = c.cfg["capacityGlobal"]
            runs.append((c.name, min(cap, SMALL_CAP), "fused", False))
            if not c.claims.get("clamped", 0):
                runs.append((c.name, LARGE_CAP, "fused", True))
    return runs


@pytest.mark.parametrize("name,cap,window,ping_pong", _runs(), ids=lambda v: str(v))
def test_surfel_case(name, cap, window, ping_pong):
    case = next(c for c in sc.small_cases() if c.name == name)
    drawn = run_case(case, cap, window, ping_pong)
    if case.kind == "splat":
        assert drawn > 0


@pytest.mark.parametrize("ping_pong", [False, True], ids=["inplace", "pingpong"])
def test_surfel_big_store_clamp(ping_pong):
    """~1.1 M surfels, count + new > capacity: the clamp on both compactions (a fresh context compacts in place)"""
    case = sc.big_cases()[0]
    run_case(case, case.cfg["capacityGlobal"], "fused", ping_pong)


def test_surfel_big_store_zero_frame():
    """~1.1 M surfels with the entry at index 0 removed and a zero-depth frame: every sub-block of the in-place compaction moves"""
    case = sc.big_cases()[1]
    run_case(case, case.cfg["capacityGlobal"], "fused", False)
