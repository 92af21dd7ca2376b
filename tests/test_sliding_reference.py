"""Sliding windows without a GPU: the row-expansion reference (tests/sliding_reference.py) reproduces the reference's
time_window.slt outputs and a scalar restatement of the Expand plan, and the engine's pane method (tumbling panes one
slide wide, each folded into k windows) equals row expansion wherever the engine accepts the query."""
import json
import os

import numpy as np
import pytest

from cnosdb_b200 import cabi
from cnosdb_b200.engine import sliding_window_grid, window_last_start
from tests.helpers import I64_MAX, I64_MIN, ReferenceError, make_query, random_arena, wrap64
from tests.sliding_reference import (expand_aggregate, n_windows_per_row, pane_aggregate, sliding_fit_grid,
                                     sliding_status)

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "time_window_slt.json")
FIELDS = ((1, cabi.TSKV_PT_I64), (2, cabi.TSKV_PT_F64))
AGGS = ("count", "sum", "min", "max", "mean")


def slt_cases():
    with open(GOLDEN) as f:
        return json.load(f)["cases"]


def slt_truth(case):
    truth = {}
    for (t, f0, f1), sid in zip(case["rows"], case["series"]):
        truth.setdefault(sid, []).append((t, f0, f1))
    out = {}
    for sid, rows in truth.items():
        ts = np.array([r[0] for r in rows], dtype=np.int64)
        ok = np.ones(ts.size, dtype=bool)
        out[sid] = [(ts, {1: (np.array([r[1] for r in rows], dtype=np.int64), ok), 2: (np.array([r[2] for r in rows]), ok)})]
    return out


def slt_queries(case):
    """[(query, {window index: row indices})]: one query per cluster of nearby windows (the 1970 / 1980 rows are ten years
    apart), restricted by a time range to the cluster's rows."""
    slide, wins = case["slide"], sorted(case["windows"], key=lambda w: w["start"])
    clusters = [[wins[0]]]
    for w in wins[1:]:
        if w["start"] - clusters[-1][-1]["start"] > 100 * slide:
            clusters.append([])
        clusters[-1].append(w)
    out = []
    for cl in clusters:
        first = cl[0]["start"]
        times = [case["rows"][r][0] for w in cl for r in w["rows"]]
        q = make_query(FIELDS, ("count", "sum"), width=case["window"], origin=case["start_time"], first_bucket_start=first,
                       n_buckets=(cl[-1]["start"] - first) // slide + 1, time_ranges=[(min(times), max(times))])
        out.append((q, {(w["start"] - first) // slide: w["rows"] for w in cl}))
    return out


@pytest.mark.parametrize("case", slt_cases(), ids=lambda c: c["name"])
def test_expansion_reproduces_the_slt_windows(case):
    truth, slide = slt_truth(case), case["slide"]
    for q, expect in slt_queries(case):
        for method in (expand_aggregate, pane_aggregate):
            got = method(truth, q, slide)
            count = got.values[got.names.index((1, "count"))]
            s0 = got.values[got.names.index((1, "sum"))].view(np.int64)
            s1 = got.values[got.names.index((2, "sum"))].view(np.float64)
            for j in range(q.n_buckets):
                rows = expect.get(j, [])
                assert count[j] == len(rows), (method.__name__, j)
                assert s0[j] == sum(case["rows"][r][1] for r in rows)
                assert s1[j] == sum(case["rows"][r][2] for r in rows)


def scalar_expansion(truth, query, slide):
    """The Expand plan with Python ints, one row copy at a time: {(group, window): (count, exact sum, min, max)} of
    column 1, or TSKV_ERR_BUCKET_RANGE."""
    w, o, fbs, nb = query.width, query.origin, query.first_bucket_start, query.n_buckets
    cmod = lambda a, b: -(abs(a) % b) if a < 0 else a % b  # noqa: E731  (truncating, b > 0)
    k = -(-w // slide)
    cells = {}
    slots = sorted(truth) if query.series_ids is None else [int(s) for s in query.series_ids]
    for slot, sid in enumerate(slots):
        for ts, cols in truth.get(sid, []):
            vals, valid = cols[1]
            for t, v, ok in zip(ts.tolist(), vals.tolist(), valid.tolist()):
                if query.time_ranges and not any(a <= t <= b for a, b in query.time_ranges):
                    continue
                last = wrap64(t - cmod(wrap64(wrap64(t - cmod(o, w)) + slide), slide))
                we0 = wrap64(last + w)
                if w % slide and not (last <= t < we0):
                    continue
                for i in range(k):
                    d = wrap64(wrap64(last - i * slide) - fbs)
                    if d < 0 or d % slide or d // slide >= nb:
                        return cabi.TSKV_ERR_BUCKET_RANGE
                    if ok:
                        key = (slot if query.group_by_series else 0, d // slide)
                        c, s, lo, hi = cells.get(key, (0, 0, v, v))
                        cells[key] = (c + 1, s + v, min(lo, v), max(hi, v))
    return cells


TRIPLES = [  # (window, slide, origin): window % slide == 0 or not, origin % window >= slide, negative origins
    (10, 5, 0), (10, 6, 0), (10, 6, 1), (10, 3, 7), (10, 3, -7), (12, 4, -25), (1000, 300, 999), (1000, 250, -1),
    (999, 333, 500), (999, 100, -998), (7, 2, 6), (7, 1, -3), (64, 64, 5), (5000, 1000, 4321), (5000, 1700, -4999),
]


def arena_for(seed, t0, step):
    rng = np.random.default_rng(seed)
    _, _, truth = random_arena(rng, n_series=5, n_points=60, fields=FIELDS, null_frac=0.2, t0=t0, step=step, jitter=step // 3)
    return truth


@pytest.mark.parametrize("t0", [1_000_000, -30 * 97])
@pytest.mark.parametrize("window,slide,origin", TRIPLES)
def test_expansion_matches_a_scalar_restatement(window, slide, origin, t0):
    truth = arena_for(window + slide, t0, 97)
    for ranges, gbs in (([], False), ([(t0 + 500, t0 + 3000)], True)):
        grid = sliding_fit_grid(truth, window, slide, origin, ranges)
        q = make_query(FIELDS, AGGS, width=window, origin=origin, first_bucket_start=grid[0], n_buckets=grid[1],
                       time_ranges=ranges, group_by_series=gbs)
        exp = scalar_expansion(truth, q, slide)
        try:
            got = expand_aggregate(truth, q, slide)
        except ReferenceError as e:
            assert exp == e.status
            continue
        assert not isinstance(exp, int), "the scalar expansion reports status %s" % exp
        count = got.values[got.names.index((1, "count"))]
        vmin = got.values[got.names.index((1, "min"))].view(np.int64)
        vmax = got.values[got.names.index((1, "max"))].view(np.int64)
        for cell in range(count.size):
            key = divmod(cell, q.n_buckets)
            c, s, lo, hi = exp.get(key, (0, 0, 0, 0))
            assert count[cell] == c, key
            if c:
                assert got.exact_sums[1][cell] == (s, c) and vmin[cell] == lo and vmax[cell] == hi, key


@pytest.mark.parametrize("t0,step", [(1_000_000, 97), (-30 * 97, 97), (-3000, 1), (I64_MIN + 5, 3), (I64_MAX - 59 * 3 - 5, 3)])
@pytest.mark.parametrize("window,slide,origin", TRIPLES)
def test_panes_folded_equal_row_expansion_where_accepted(window, slide, origin, t0, step):
    """The design without a GPU: wherever the engine accepts the query, folding panes gives what row expansion gives
    (bit for bit: the same rows land in the same windows), including the row that falls off a grid one window short."""
    truth = arena_for(window * 7 + slide, t0, step)
    grid = sliding_fit_grid(truth, window, slide, origin, [])
    assert grid is not None
    for fbs, nb in (grid, (grid[0] + slide, grid[1] - 1), (grid[0], grid[1] - 1)):
        q = make_query(FIELDS, AGGS, width=window, origin=origin, first_bucket_start=fbs, n_buckets=nb)
        if sliding_status(truth, q, slide) is not None:
            continue
        res = []
        for method in (expand_aggregate, pane_aggregate):
            try:
                res.append(method(truth, q, slide))
            except ReferenceError as e:
                res.append(e.status)
        a, b = res
        if isinstance(a, int) or isinstance(b, int):
            assert a == b
            continue
        assert (a.validity == b.validity).all() and (a.values == b.values).all()


def test_refusals_follow_the_library_order():
    truth = arena_for(3, -30 * 97, 97)  # rows on both sides of the truncating-% regime
    grid = lambda w, s: sliding_fit_grid(truth, w, s, 0, [])  # noqa: E731
    q = lambda w, aggs=AGGS, nb=None, **kw: make_query(FIELDS, aggs, width=w, origin=0, first_bucket_start=grid(w, 5)[0],  # noqa: E731
                                                       n_buckets=nb or grid(w, 5)[1], **kw)
    assert sliding_status(truth, q(10), 0) == cabi.TSKV_ERR_INVALID_ARG
    assert sliding_status(truth, q(10, ("count", "first")), 10) is None          # slide == window: the tumbling scan
    assert sliding_status(truth, q(10, ("count", "last")), 5) == cabi.TSKV_ERR_UNSUPPORTED
    assert sliding_status(truth, q(10), 11) == cabi.TSKV_ERR_UNSUPPORTED
    assert sliding_status(truth, make_query(FIELDS, AGGS, width=2**61, first_bucket_start=0, n_buckets=4), 2**60) == \
        cabi.TSKV_ERR_UNSUPPORTED
    assert sliding_status(truth, q(505), 5) == cabi.TSKV_ERR_INVALID_ARG          # k = 101
    assert sliding_status(truth, q(500, nb=99), 5) == cabi.TSKV_ERR_INVALID_ARG   # n_buckets < k
    assert sliding_status(truth, q(10), 5) is None                                # window % slide == 0: any regime
    assert sliding_status(truth, q(10), 6) == cabi.TSKV_ERR_UNSUPPORTED           # truncating rows, 10 % 6 != 0
    assert sliding_status(truth, q(10, time_ranges=[(0, 10**6)]), 6) is None      # ... not selected


def test_window_grid_helper():
    for window, slide, origin in TRIPLES:
        for lo, hi in ((0, 0), (12_345, 99_999), (10**12, 10**12 + 7)):
            fbs, nb = sliding_window_grid(lo, hi, window, slide, origin)
            k = n_windows_per_row(window, slide)
            assert fbs == window_last_start(lo, window, slide, origin) - (k - 1) * slide
            assert fbs + (nb - 1) * slide == window_last_start(hi, window, slide, origin)
            truth = {0: [(np.array([lo, hi], dtype=np.int64), {})]}
            assert sliding_fit_grid(truth, window, slide, origin, []) == (fbs, nb)
    assert window_last_start(I64_MIN + 2, 10, 3, 7) == wrap64(I64_MIN + 2 - (wrap64(I64_MIN + 2 - 7 + 3) % 3))  # wrapped up
