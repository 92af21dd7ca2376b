"""Exact per-cell co-moments of column pairs (tskv_query.n_pairs) for arenas described by a `truth` dict (tests/helpers.py
random_arena's: truth[series] = [(ts, {column: (values, valid)}), ...] per column group).

The row selection is restated row by row, so that x and y stay paired: a row counts when its series is selected, its
timestamp lies in the query's time ranges and in a bucket of the grid (or of the edges), the AND-ed predicates hold, no
row-drop tombstone covers it, and both x and y are valid and not masked by a column tombstone. A column group without x
or y has no paired row. Overlapping chunk files (`files=`) are merged as helpers.exact_aggregate merges them, with x and
y as the merge's columns: predicates and row drops before the merge, the time ranges, column tombstones and buckets on
the merged rows. Per cell: n, C = sum (x - mx)(y - my), M2x and M2y over the paired rows, computed exactly over the
values converted to f64 and rounded once (NaN with a NaN or infinite value)."""
import copy
import math
import os

import numpy as np

from cnosdb_b200.engine import PushedAggregate
from tests import helpers


def exact_comoments(xs, ys):
    """(n, C, M2x, M2y) of paired f64 values, exactly, each rounded once (n == 0: Nones)."""
    n = len(xs)
    if n == 0:
        return 0, None, None, None
    xs, ys = [float(v) for v in xs], [float(v) for v in ys]
    if not all(math.isfinite(v) for v in xs + ys):
        bad_x = not all(math.isfinite(v) for v in xs)
        bad_y = not all(math.isfinite(v) for v in ys)
        return n, math.nan, (math.nan if bad_x else _m2(xs)), (math.nan if bad_y else _m2(ys))
    (kx, qx), (ky, qy) = _scaled(xs), _scaled(ys)
    return n, _co(kx, qx, ky, qy), _co(kx, qx, kx, qx), _co(ky, qy, ky, qy)


def _m2(vs):
    k, q = _scaled(vs)
    return _co(k, q, k, q)


def _scaled(vs):
    """f64 values as integers k over one common power-of-two denominator q: v = k / q exactly."""
    ratios = [v.as_integer_ratio() for v in vs]
    q = max(d for _, d in ratios)
    return [p * (q // d) for p, d in ratios], q


def _co(ka, qa, kb, qb):
    """sum (a - ma)(b - mb) = (n sum ka kb - sum ka sum kb) / (n qa qb), rounded once (int / int rounds correctly)."""
    n = len(ka)
    num = n * sum(a * b for a, b in zip(ka, kb)) - sum(ka) * sum(kb)
    try:
        return num / (n * qa * qb)
    except OverflowError:
        return math.inf if num > 0 else -math.inf


def paired_rows(truth, query, pair, tombstones=None, group_ids=None, edges=None, labels=None, files=None):
    """{cell: ([x], [y])} of the pair (x_id, x_pt, y_id, y_pt) under `query` (a QueryOption); cell = group * n_buckets +
    bucket, group = series slot (group_by_series), group_ids[slot] (GROUP BY tags) or 0. files: the file id of every
    column group in truth's order (helpers.exact_aggregate's `files`)."""
    x_id, x_pt, y_id, y_pt = pair
    glob, rows_t, cols_t = helpers.tombstone_lists(tombstones)
    file_of = helpers.files_by_series(truth, files)
    mq = copy.copy(query)  # the merge's query columns: the operands
    mq.columns = [PushedAggregate(x_id, x_pt, 0), PushedAggregate(y_id, y_pt, 0)]
    ops = list(dict.fromkeys((x_id, y_id)))
    sel = list(query.series_ids) if query.series_ids is not None else sorted(truth)
    cells, xs, ys = [], [], []
    for slot, sid in enumerate(sel):
        sid = int(sid)
        if sid not in truth:
            continue
        cgs = truth[sid]
        group = slot if query.group_by_series else (int(group_ids[slot]) if group_ids is not None else 0)
        row_drop = glob + rows_t.get(sid, [])
        units = []  # (timestamps, columns, rows that pass the predicates and row drops)
        for streams in helpers.overlap_groups(cgs, file_of.get(sid)):
            if len(streams) >= 2:
                ts, cols = helpers._merged_rows(cgs, streams, mq, ops, row_drop)
                cols = {c: (v.view(helpers._typed(pt, []).dtype), ok) for (c, pt), (v, ok) in
                        zip(((x_id, x_pt), (y_id, y_pt)), (cols[x_id], cols[y_id]))}
                units.append((ts, cols, np.ones(ts.size, dtype=bool)))
                continue
            for k in streams[0]:
                ts, cols = cgs[k]
                if x_id not in cols or y_id not in cols:
                    continue
                ts = np.asarray(ts, dtype=np.int64)
                units.append((ts, cols, helpers._predicates_hold(query, ts, cols) & ~helpers._in_ranges(ts, row_drop)))
        for ts, cols, keep in units:
            if query.time_ranges:
                keep = keep & helpers._in_ranges(ts, query.time_ranges)
            (xv, xok), (yv, yok) = cols[x_id], cols[y_id]
            keep &= np.asarray(xok, dtype=bool) & np.asarray(yok, dtype=bool)
            keep &= ~helpers._in_ranges(ts, cols_t.get((sid, x_id), []))
            keep &= ~helpers._in_ranges(ts, cols_t.get((sid, y_id), []))
            if edges is not None:
                e = np.asarray(edges, dtype=np.int64)
                b = np.searchsorted(e, ts, side="right") - 1
                inb = (ts >= e[0]) & (ts < e[-1])
                if labels is not None:
                    b = np.where(inb, np.asarray(labels)[np.clip(b, 0, len(labels) - 1)], 0)
            else:
                b, inb = helpers.bucket_index(ts, query)
            keep &= inb
            cells.append(group * query.n_buckets + np.asarray(b, dtype=np.int64)[keep])
            # (int64 / uint64 / float64 arrays: astype is (double)x, round to nearest)
            xs.append(np.asarray(xv).astype(np.float64)[keep])
            ys.append(np.asarray(yv).astype(np.float64)[keep])
    if not cells:
        return {}
    cl = np.concatenate(cells)
    order = np.argsort(cl, kind="stable")  # (a cell's rows keep their order)
    cl, fx, fy = cl[order], np.concatenate(xs)[order], np.concatenate(ys)[order]
    heads = np.flatnonzero(np.concatenate([[True], cl[1:] != cl[:-1]])) if cl.size else cl
    bounds = list(heads) + [cl.size]
    return {int(cl[a]): (fx[a:z].tolist(), fy[a:z].tolist()) for a, z in zip(bounds[:-1], bounds[1:])}


def exact_pair_cells(truth, query, pair, n_cells, **kw):
    """Arrays n [u64], C, M2x, M2y [f64; NaN where n == 0] over n_cells cells."""
    n = np.zeros(n_cells, dtype=np.uint64)
    c, m2x, m2y = (np.full(n_cells, np.nan) for _ in range(3))
    for cell, (xs, ys) in paired_rows(truth, query, pair, **kw).items():
        n[cell], c[cell], m2x[cell], m2y[cell] = exact_comoments(xs, ys)
    return n, c, m2x, m2y


def check_pair(res, k, exact, rtol=1e-9, what=""):
    """The scan's raw outputs of pair k against exact_pair_cells: n exactly; M2x / M2y within rtol of their own value; C
    within rtol of the larger of |C| and the cell's sqrt(M2x M2y) (C may cancel to 0, and |C| <= sqrt(M2x M2y)); NaN where
    the reference is NaN; validity iff n >= 1."""
    n_e, c_e, x_e, y_e = exact
    n, nok = res.pair(k, "n")
    assert nok.all(), what
    np.testing.assert_array_equal(n.ravel(), n_e, err_msg=what + " n")
    for name, e in (("c", c_e), ("m2x", x_e), ("m2y", y_e)):
        v, ok = res.pair(k, name)
        v, ok = v.ravel(), ok.ravel()
        np.testing.assert_array_equal(ok, n_e > 0, err_msg=what + " validity " + name)
        m = n_e > 0
        with np.errstate(invalid="ignore"):
            scale = np.nan_to_num(np.sqrt(np.abs(x_e * y_e)), nan=0.0) if name == "c" else 0.0
            bound = rtol * np.maximum(np.abs(e), scale) + 1e-300
        for i in np.nonzero(m)[0]:
            if math.isnan(e[i]):
                assert math.isnan(v[i]), (what, name, i, v[i])
            else:
                assert abs(v[i] - e[i]) <= bound[i], (what, name, i, v[i], e[i])


# ---- the reference's covar / corr goldens (tests/golden/covar_slt.json, written by tests/golden/make_covar_golden.py) ----
GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "covar_slt.json")
TB2_TYPES = {"f0": "u64", "f1": "f64", "f4": "i64"}  # the numeric fields of func_tb2 (f2 BOOLEAN, f3 STRING)


def load_golden():
    import json
    with open(GOLDEN) as f:
        return json.load(f)


def tb2_column(g, name):
    """A func_tb2 operand as an int64 / uint64 / float64 array in row order; `-f1` is f1 negated (the planner's
    expression, stored as a column of its own for the scan)."""
    rows = g["tables"]["func_tb2"]["rows"]
    cols = g["tables"]["func_tb2"]["columns"]
    neg = name.startswith("-")
    base = name.lstrip("-")
    vals = [r[cols.index(base)] for r in rows]
    kind = TB2_TYPES[base]
    a = np.array([float(v) for v in vals]) if kind == "f64" else np.array([int(v) for v in vals],
                                                                        dtype=np.uint64 if kind == "u64" else np.int64)
    return -a if neg else a
