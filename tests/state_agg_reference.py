"""Exact per-cell compact_state_agg(time, x) (TSKV_QUERY_N_STATE_AGGS) for arenas described by a `truth` dict (tests/helpers.py
random_arena's).

The row selection restates covariance_reference.paired_rows with one operand, except that NULL values are kept: series,
time ranges, buckets, predicates and row tombstones select a row; a NULL in the page's bitmap, a column tombstone over the
row or a merged row of an overlap merge group without a value of the operand make the row's state NULL (None here).

`fold` restates the reference's DurationStates (state_agg_data.rs): `handle_record` adds t' - t to the duration of the
earlier point's state for every pair of consecutive points, and `finalize` gives the last point's state a 0 entry when it
has none. The accumulator's `evaluate` sorts every row of the cell by time and skips rows with a NULL time
(state_agg_accumulator.rs); `update_batch_reference` restates that over a split of the rows into batches."""
import copy
import json
import os

import numpy as np

from cnosdb_b200 import cabi
from cnosdb_b200.engine import PushedAggregate
from tests import helpers


def fold(points):
    """DurationStates::handle_record over points [(t, state)] in time order, then finalize -> {state: duration}."""
    durations, last = {}, None
    for t, s in points:
        if last is not None:
            ls, lt = last
            durations[ls] = durations.get(ls, 0) + (t - lt)
        last = (s, t)
    if last is not None:
        durations.setdefault(last[0], 0)
    return durations


def update_batch_reference(rows, cuts):
    """CompactStateAggAccumulator: update_batch appends every row of the batches rows[cuts[i]:cuts[i + 1]] ((t or None,
    state)), evaluate sorts them by time, skips NULL times and folds -> {state: duration}."""
    kept = []
    for a, b in zip(cuts[:-1], cuts[1:]):
        kept.extend(rows[a:b])
    kept = sorted((r for r in kept if r[0] is not None), key=lambda r: r[0])
    return fold(kept)


def _typed_state(v, pt):
    return int(np.int64(v)) if pt == cabi.TSKV_PT_I64 else int(np.uint64(v))


def selected_points(truth, query, col, pt, tombstones=None, group_ids=None, edges=None, files=None):
    """{cell: [(t, state)]} of operand (col, pt) under `query`, each cell's points in time order (a cell holds one series:
    its times are distinct). state is the typed value, None for a NULL."""
    glob, rows_t, cols_t = helpers.tombstone_lists(tombstones)
    file_of = helpers.files_by_series(truth, files)
    mq = copy.copy(query)  # the merge's query column: the operand
    mq.columns = [PushedAggregate(col, pt, 0)]
    sel = list(query.series_ids) if query.series_ids is not None else sorted(truth)
    out = {}
    for slot, sid in enumerate(sel):
        sid = int(sid)
        if sid not in truth:
            continue
        cgs = truth[sid]
        group = slot if query.group_by_series else (int(group_ids[slot]) if group_ids is not None else 0)
        row_drop = glob + rows_t.get(sid, [])
        units = []  # (timestamps, (values, validity), rows that pass the predicates and row drops)
        for streams in helpers.overlap_groups(cgs, file_of.get(sid)):
            if len(streams) >= 2:
                ts, cols = helpers._merged_rows(cgs, streams, mq, [col], row_drop)
                units.append((ts, cols[col], np.ones(ts.size, dtype=bool)))
                continue
            for k in streams[0]:
                ts, cols = cgs[k]
                if col not in cols:  # (the scan refuses such a group where it can hold selected rows)
                    continue
                ts = np.asarray(ts, dtype=np.int64)
                units.append((ts, cols[col], helpers._predicates_hold(query, ts, cols) & ~helpers._in_ranges(ts, row_drop)))
        for ts, (v, ok), keep in units:
            if query.time_ranges:
                keep = keep & helpers._in_ranges(ts, query.time_ranges)
            null = ~np.asarray(ok, dtype=bool) | helpers._in_ranges(ts, cols_t.get((sid, col), []))
            if edges is not None:
                e = np.asarray(edges, dtype=np.int64)
                b = np.searchsorted(e, ts, side="right") - 1
                inb = (ts >= e[0]) & (ts < e[-1])
            else:
                b, inb = helpers.bucket_index(ts, query)
            keep = keep & inb
            v = np.asarray(v)
            for i in np.flatnonzero(keep):
                cell = group * query.n_buckets + int(b[i])
                out.setdefault(cell, []).append((int(ts[i]), None if null[i] else _typed_state(v[i], pt)))
    return {c: sorted(p, key=lambda x: x[0]) for c, p in out.items()}


def exact_state_maps(truth, query, col, pt, n_cells, **kw):
    """[{state: duration}] per cell (an empty map for a cell without rows)."""
    pts = selected_points(truth, query, col, pt, **kw)
    return [fold(pts.get(c, [])) for c in range(n_cells)]


def check_state_maps(res, col, exact, what=""):
    """ScanResult `res`'s maps and entry counts of state agg column `col` against exact_state_maps, as maps."""
    got = [m for row in res.state_maps(col) for m in row]
    assert len(got) == len(exact), what
    bad = [(c, got[c], exact[c]) for c in range(len(exact)) if got[c] != exact[c]]
    assert not bad, (what, bad[:3])
    n, ok = res.column(col, "state_entries")
    assert ok.all(), what
    np.testing.assert_array_equal(n.reshape(-1), np.array([len(m) for m in exact], dtype=np.uint64), err_msg=what)


# ---- the reference's answers (tests/golden/compact_state_agg_slt.json, written by make_compact_state_agg_golden.py) ----
GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "compact_state_agg_slt.json")


def load_golden():
    with open(GOLDEN) as f:
        return json.load(f)
