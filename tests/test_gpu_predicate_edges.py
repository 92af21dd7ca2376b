"""Pushed field predicates with constants at the page statistics' bounds. Predicate columns of i64, u64 and f64 (simple8b,
constant run-length, raw and Gorilla pages; single-row, all-null, all-NaN and all -0.0 pages, NaN next to a page's
minimum or maximum, a column some column groups lack) are compared with every page's exact minimum and maximum, one step
beyond each, the type limits, +-0.0, a subnormal and NaNs of both signs, under each source of page statistics: the
device's own (k_page_stats), the caller's (exact, with NaN or -0.0 bounds or min > max, loose), a host-resident page set
with the caller's, and none. Results must equal the exact reference bit for bit and each other across the sources, and
pruned_page_count must equal a count restated here from the generated arrays: a column group is skipped when the
bounds of one of its predicate pages leave no value that can satisfy the comparison, and only then."""
import math
import os
import subprocess
import sys

import numpy as np
import pytest

from cnosdb_b200 import cabi, datagen
from oracle import pyoracle as orc
from tests.helpers import I64_MAX, I64_MIN, assert_matches_exact, exact_aggregate, make_query

pytestmark = pytest.mark.gpu

T0, STEP = 5_000_000, 1000
N_SERIES = 48
AGG_FIELDS = ((1, cabi.TSKV_PT_I64), (2, cabi.TSKV_PT_F64))
AGGS = ("count", "sum", "min", "max", "mean")
PRED = {cabi.TSKV_PT_I64: 10, cabi.TSKV_PT_U64: 11, cabi.TSKV_PT_F64: 12}  # predicate column of each type
OPS = ("==", "!=", "<", "<=", ">", ">=")
MAX_PREDICATES = 8  # TSKV_MAX_PREDICATES
# the pages whose bounds become constants: the single-row ones, NaN next to the bounds, inf / subnormals / +-0.0
BOUND_SAMPLE = {0, 8, 16, 24, 32, 40, 2, 9, 3, 10, 4, 11, 17, 21}
NEG_NAN, POS_NAN = np.uint64(0xFFF8000000000001).view(np.float64), np.uint64(0x7FF0000000000002).view(np.float64)


def _pred_values(rng, pt, sid, n):
    """(values, validity, encoder) of one predicate page."""
    valid = np.ones(n, dtype=bool)
    if sid % 9 == 4:
        valid[:] = False                       # all null
    elif sid % 5 == 2:
        valid = rng.random(n) >= 0.3
    enc = None
    if pt == cabi.TSKV_PT_F64:
        v = np.cumsum(rng.integers(-40, 41, n)).astype(np.float64) * 0.25 + rng.integers(-3, 4) * 10.0
        k = sid % 7
        if k == 0:
            v[:] = np.where(rng.random(n) < 0.5, NEG_NAN, POS_NAN)            # all NaN
        elif k == 1:
            v[:] = -0.0                                                       # all -0.0
        elif k == 2 and n >= 3:                                               # NaN next to the minimum and the maximum
            for i in (int(np.argmin(v)), int(np.argmax(v))):
                v[i - 1 if i else i + 1] = NEG_NAN if i % 2 else POS_NAN
        elif k == 3:
            v[rng.integers(0, n)] = [np.inf, -np.inf, 5e-324, -0.0][sid % 4]
        elif k == 4:
            v = rng.choice([-0.0, 0.0, 5e-324, -5e-324, 2.2250738585072014e-308], n)
        enc = datagen.encode_raw if sid % 2 else None                         # raw or Gorilla
        return v, valid, enc
    if pt == cabi.TSKV_PT_U64:
        base = [0, 2**63 - 50, 2**64 - 500, 1000][sid % 4]
        v = (np.uint64(base) + np.cumsum(rng.integers(0, 3, n)).astype(np.uint64))
    else:
        base = [I64_MIN, -500, 0, I64_MAX - 700][sid % 4]
        v = np.int64(base) + np.cumsum(rng.integers(0, 4, n)).astype(np.int64)
    k = sid % 3
    if k == 1:
        v[:] = v[0]                            # constant: a run-length page
    elif k == 2:
        enc = datagen.encode_raw
    return v, valid, enc


def predicate_arena(seed):
    """-> (arena, descs, truth). Series 8k hold one row; series 0, 6, 12, ... lack the u64 column; series 5 has a
    second column group without any predicate column."""
    rng = np.random.default_rng(seed)
    b = datagen.ArenaBuilder()
    truth = {}
    for sid in range(N_SERIES):
        n = 1 if sid % 8 == 0 else int(rng.integers(20, 200))
        ts = T0 + np.arange(n, dtype=np.int64) * STEP
        iv = np.cumsum(rng.integers(-50, 51, n)).astype(np.int64)
        fv = np.cumsum(rng.integers(-3, 4, n)).astype(np.float64) + rng.random(n)
        ok = np.ones(n, dtype=bool)
        fl = [(1, cabi.TSKV_PT_I64, iv, None), (2, cabi.TSKV_PT_F64, fv, None)]
        cols = {1: (iv, ok), 2: (fv, ok)}
        for pt, c in PRED.items():
            if pt == cabi.TSKV_PT_U64 and sid % 6 == 0:
                continue
            v, valid, enc = _pred_values(rng, pt, sid, n)
            fl.append((c, pt, v, None if valid.all() else valid, enc) if enc else (c, pt, v, None if valid.all() else valid))
            cols[c] = (v, valid)
        b.add_column_group(sid, ts, fl)
        truth[sid] = [(ts, cols)]
        if sid == 5:
            ts2 = T0 + (n + np.arange(10, dtype=np.int64)) * STEP
            v2 = np.arange(10, dtype=np.int64)
            b.add_column_group(sid, ts2, [(1, cabi.TSKV_PT_I64, v2, None), (2, cabi.TSKV_PT_F64, v2.astype(np.float64), None)])
            truth[sid].append((ts2, {1: (v2, np.ones(10, dtype=bool)), 2: (v2.astype(np.float64), np.ones(10, dtype=bool))}))
    arena, descs = b.finish()
    return arena, descs, truth


# ---- the statistics, restated from the generated arrays ----------------------------------------------------------------

def page_bounds(pt, values, valid):
    """Numeric (min, max) of a page's non-null, non-NaN values (-0.0 counts as +0.0), or None when it has none."""
    v = np.asarray(values)[np.asarray(valid, dtype=bool)]
    if pt == cabi.TSKV_PT_F64:
        v = v[~np.isnan(v)]
        if v.size == 0:
            return None
        return float(v.min()) + 0.0, float(v.max()) + 0.0
    if v.size == 0:
        return None
    return int(v.min()), int(v.max())


def rules_out(pt, op, c, bounds):
    """Can no value in the closed interval `bounds` satisfy `value <op> c`? bounds: (min, max), None (no value: nothing
    is ever TRUE) or "unknown": any value of the type (an integer compared with a limit of its type can still be ruled
    out; an f64 page without bounds may hold NaNs of either sign, so only a NaN constant rules it out)."""
    if isinstance(c, float) and math.isnan(c):
        return True
    if bounds is None:
        return True
    if bounds == "unknown":
        if pt == cabi.TSKV_PT_F64:
            return False
        bounds = (0, 2**64 - 1) if pt == cabi.TSKV_PT_U64 else (I64_MIN, I64_MAX)
    mn, mx = bounds
    return {"==": c < mn or c > mx, "!=": mn == mx == c, "<": mn >= c, "<=": mn > c, ">": mx <= c, ">=": mx < c}[op]


def expected_pruned(truth, preds, stats):
    """Field pages of the query columns in column groups that some predicate's page statistics rule out. stats:
    {(sid, cg index, column): bounds} or None (no statistics at all)."""
    if stats is None:
        return 0
    n = 0
    for sid, cgs in truth.items():
        for g, (_, cols) in enumerate(cgs):
            if any(c in cols and rules_out(pt, op, v, stats[(sid, g, c)]) for c, pt, op, v in preds):
                n += sum(1 for c, _ in AGG_FIELDS if c in cols)
    return n


def stats_table(descs, truth, kind):
    """(VALUE_STATS_DTYPE array for set_value_stats, {(sid, cg, column): bounds} the scan then prunes with).
    kind: "exact" (pages without a value: no statistics), "odd" (NaN bounds for pages that hold a NaN, -0.0 for zero
    bounds, min > max for pages without a value), "loose" (bounds a few steps wider)."""
    st = np.zeros(len(descs), dtype=cabi.VALUE_STATS_DTYPE)
    eff = {}
    cg_of = {}
    for i, d in enumerate(descs):
        sid, col, pt = int(d["series_id"]), int(d["column_id"]), int(d["phys_type"])
        if pt == cabi.TSKV_PT_TIME:
            cg_of[sid] = cg_of.get(sid, -1) + 1
            continue
        g = cg_of[sid]
        values, valid = truth[sid][g][1][col]
        bnd = page_bounds(pt, values, valid)
        has_nan = pt == cabi.TSKV_PT_F64 and bool(np.isnan(np.asarray(values)[valid]).any())
        enc = (lambda x: np.uint64(np.float64(x).view(np.uint64))) if pt == cabi.TSKV_PT_F64 else \
            (lambda x: np.uint64(x & 0xFFFFFFFFFFFFFFFF))
        if bnd is None:
            if kind == "odd":
                st[i] = (enc(1), enc(0), cabi.TSKV_STATS_MINMAX, 0)  # min > max: no value
            eff[(sid, g, col)] = None if kind == "odd" else "unknown"
            continue
        mn, mx = bnd
        if kind == "odd" and has_nan:
            st[i] = (enc(mn), np.uint64(0x7FF8000000000000), cabi.TSKV_STATS_MINMAX, 0)
            eff[(sid, g, col)] = "unknown"
            continue
        if kind == "odd" and pt == cabi.TSKV_PT_F64:
            mn, mx = (-0.0 if mn == 0 else mn), (-0.0 if mx == 0 else mx)
        if kind == "loose":
            if pt == cabi.TSKV_PT_F64:
                mn, mx = np.nextafter(np.nextafter(mn, -np.inf), -np.inf), np.nextafter(mx, np.inf)
                mn, mx = float(mn) + 0.0, float(mx) + 0.0
            elif pt == cabi.TSKV_PT_U64:
                mn, mx = max(mn - 3, 0), min(mx + 2, 2**64 - 1)
            else:
                mn, mx = max(mn - 3, I64_MIN), min(mx + 2, I64_MAX)
        st[i] = (enc(mn), enc(mx), cabi.TSKV_STATS_MINMAX, 0)
        eff[(sid, g, col)] = (mn + 0.0, mx + 0.0) if pt == cabi.TSKV_PT_F64 else (mn, mx)
    return st, eff


def device_stats(truth):
    """What k_page_stats computes: the exact bounds, None for pages without a value."""
    return {(sid, g, c): page_bounds(pt, *cols[c]) for sid, cgs in truth.items() for g, (_, cols) in enumerate(cgs)
            for c, pt in [(1, cabi.TSKV_PT_I64), (2, cabi.TSKV_PT_F64)] + [(c, pt) for pt, c in PRED.items()] if c in cols}


# ---- the queries ---------------------------------------------------------------------------------------------------------

def _step(pt, x, d):
    if pt == cabi.TSKV_PT_F64:
        return float(np.nextafter(x, np.inf if d > 0 else -np.inf))
    lo, hi = (0, 2**64 - 1) if pt == cabi.TSKV_PT_U64 else (I64_MIN, I64_MAX)
    return min(max(x + d, lo), hi)


def constants(pt, truth):
    col = PRED[pt]
    cs = set()
    for sid, cgs in truth.items():
        for _, cols in cgs:
            if col in cols:
                bnd = page_bounds(pt, *cols[col])
                if bnd is not None and sid in BOUND_SAMPLE:
                    for x in bnd:
                        cs.update({x, _step(pt, x, -1), _step(pt, x, 1)})
    if pt == cabi.TSKV_PT_F64:
        cs.update({math.inf, -math.inf, float(np.finfo(np.float64).max), -float(np.finfo(np.float64).max), 0.0, 5e-324,
                   -5e-324})
        out = sorted(cs) + [-0.0, NEG_NAN, POS_NAN]
    elif pt == cabi.TSKV_PT_U64:
        out = sorted(cs | {0, 1, 2**63 - 1, 2**63, 2**63 + 1, 2**64 - 1})
    else:
        out = sorted(cs | {I64_MIN, I64_MIN + 1, -1, 0, 1, I64_MAX - 1, I64_MAX})
    return out


def predicate_sets(truth):
    """Single predicates of every op x type x constant, then AND-ed sets of up to TSKV_MAX_PREDICATES."""
    rng = np.random.default_rng(3)
    out = []
    per_type = {pt: constants(pt, truth) for pt in PRED}
    for pt, cs in per_type.items():
        for c in cs:
            for op in OPS:
                out.append([(PRED[pt], pt, op, c)])
    for k in range(40):
        m = int(rng.integers(2, MAX_PREDICATES + 1))
        ps = [(1, cabi.TSKV_PT_I64, str(rng.choice(OPS)), int(rng.integers(-300, 300)))]  # the aggregated column itself
        for _ in range(m - 1):
            pt = list(PRED)[int(rng.integers(0, 3))]
            cs = per_type[pt]
            ps.append((PRED[pt], pt, str(rng.choice(OPS)), cs[int(rng.integers(0, len(cs)))]))
        out.append(ps)
    return out


def _query(preds):
    return make_query(AGG_FIELDS, AGGS, group_by_series=True, predicates=preds)


# ---- the statistics source without any statistics (TSKV_NO_VALUE_STATS, read once per process) -------------------------

def _scan_all_without_value_stats(out_path):
    from cnosdb_b200.engine import Engine
    arena, descs, truth = predicate_arena(11)
    e = Engine(0)
    pages = e.upload_pages(arena, descs)
    vals, valid, pruned = [], [], []
    for preds in predicate_sets(truth):
        r = e.scan_aggregate(pages, _query(preds))
        vals.append(r.values)
        valid.append(r.validity)
        pruned.append(e.counters()["pruned_page_count"])
    pages.close()
    e.close()
    np.savez(out_path, values=np.stack(vals), validity=np.stack(valid), pruned=np.array(pruned))


def _results_equal(a, b, what):
    """COUNT / integer SUM / MIN / MAX / MEAN bit for bit (an f64 sum depends on the order)."""
    for j, (col, agg) in enumerate(a.names):
        if col == 2 and agg in ("sum", "mean"):
            continue
        assert (a.validity[j] == b.validity[j]).all() and (a.values[j] == b.values[j]).all(), "%s: col %s %s" % (what, col, agg)


def test_predicates_at_statistics_bounds(engine, tmp_path):
    arena, descs, truth = predicate_arena(11)
    env = dict(os.environ, TSKV_NO_VALUE_STATS="1")
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    out = str(tmp_path / "no_stats.npz")
    subprocess.check_call([sys.executable, "-c", "import sys; sys.path.insert(0, %r); from tests import test_gpu_predicate_edges as t; "
                           "t._scan_all_without_value_stats(%r)" % (root, out)], env=env, cwd=root)
    no_stats = np.load(out)

    dev = engine.upload_pages(arena, descs)                       # k_page_stats
    caller = {k: engine.upload_pages(arena, descs) for k in ("exact", "odd", "loose")}
    effective = {"device": device_stats(truth), "host_none": None}
    for k, p in caller.items():
        st, effective[k] = stats_table(descs, truth, k)
        p.set_value_stats(st)
    host = engine.upload_pages(arena, descs, host_resident=True)
    host_none = engine.upload_pages(arena, descs, host_resident=True)
    st, effective["host"] = stats_table(descs, truth, "exact")
    host.set_value_stats(st)
    sources = [("device", dev), ("exact", caller["exact"]), ("odd", caller["odd"]), ("loose", caller["loose"]),
               ("host", host), ("host_none", host_none)]

    n_pruned = {k: 0 for k, _ in sources}
    for i, preds in enumerate(predicate_sets(truth)):
        q = _query(preds)
        exp = exact_aggregate(truth, q)
        _, pts = orc.scan_aggregate(arena, descs, q, return_points=True)
        orc.set_value_stats_pruning(False)
        try:
            _, pts_all = orc.scan_aggregate(arena, descs, q, return_points=True)
        finally:
            orc.set_value_stats_pruning(True)
        first = None
        for name, pages in sources:
            what = "%s %s" % (name, preds)
            got = engine.scan_aggregate(pages, q)
            c = engine.counters()
            assert_matches_exact(got, exp, what=what)
            want = expected_pruned(truth, preds, effective[name])
            assert c["pruned_page_count"] == want, "%s: %d pages pruned, expected %d" % (what, c["pruned_page_count"], want)
            n_pruned[name] += want
            if name == "device":
                assert c["points_decoded"] == pts, "%s: points %d, oracle %d" % (what, c["points_decoded"], pts)
            if name == "host_none":
                assert c["points_decoded"] == pts_all, "%s: points %d, oracle %d" % (what, c["points_decoded"], pts_all)
            if first is None:
                first = got
            else:
                _results_equal(got, first, what)
        assert int(no_stats["pruned"][i]) == 0, preds
        nv = type("R", (), {"names": first.names, "values": no_stats["values"][i], "validity": no_stats["validity"][i]})
        _results_equal(nv, first, "TSKV_NO_VALUE_STATS=1 %s" % (preds,))
    assert all(n_pruned[k] > 0 for k in ("device", "exact", "odd", "loose", "host")), n_pruned
    for p in [dev, host, host_none] + list(caller.values()):
        p.close()
