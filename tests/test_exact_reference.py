"""The exact reference of tests/helpers.py checked on its own (no GPU): its window arithmetic against the reference's
known-answer vectors and the oracle's restatement, and its aggregates against the oracle on every arena of the bucket
geometry sweep and of tests/exact_arenas.py (FIRST / LAST runs, tombstones, the overlap merge), plus hand-worked cases.
COUNT / SUM / MIN / MAX / FIRST / LAST must agree bit for bit; f64 sums within the order-free bound; the integer MEAN is
not compared (the oracle keeps an f64 running sum, the reference the exact one)."""
import math

import numpy as np
import pytest

from oracle import pyoracle as orc
from tests.helpers import (DBL_MAX, F64_LENGTHS, GEOMETRY_CASES, I64_MAX, I64_MIN, OrderDependentSum, ReferenceError,
                           assert_matches_exact, ceil_sliding_window, exact_aggregate, f64_edge_arena, f64_edge_expected,
                           f64_edge_queries, f64_sum_class, floor_sliding_window, geometry_arena, geometry_queries,
                           geometry_ranges, make_query, raw_key_edge, sel_unsupported, sliding_window, split_ranges)
from tests import exact_arenas as ea
from cnosdb_b200 import cabi, datagen


def test_window_known_answers(golden):
    cases = golden["window_kat"]["cases"]
    assert len(cases) == 14
    for c in cases:
        f = ceil_sliding_window if c["ceil"] else floor_sliding_window
        assert f(c["t"], c["window"], c["slide"], c["start_time"]) == (c["start"], c["end"]), c


EDGE_T = [I64_MIN, I64_MIN + 1, -2**62 - 1, -2**62, -7, -1, 0, 1, 6, 2**62 - 1, 2**62, I64_MAX - 1, I64_MAX]
EDGE_W = [1, 2, 3, 7, 1000, 2**33 + 5, 2**61 - 1, 2**61, 2**62 + 1, I64_MAX]
EDGE_O = [0, 5, -5, 1001, I64_MIN, I64_MAX, -2**62]


def test_sliding_window_matches_oracle_on_edges():
    for w in EDGE_W:
        for o in EDGE_O:
            ts = np.array(EDGE_T, dtype=np.int64)
            ws, we = sliding_window(ts, w, w, o)
            for k, t in enumerate(EDGE_T):
                exp = orc.sliding_window(t, w, w, o)
                assert (int(ws[k]), int(we[k])) == exp, (t, w, o)
                assert sliding_window(t, w, w, o) == exp


def test_integer_sum_and_mean_are_exact():
    """Values whose wrapping sum and f64 running sum are both wrong: S is a Python int, MEAN = float(S) / float(n)."""
    v = np.array([I64_MAX, I64_MAX, I64_MIN, 5, I64_MAX], dtype=np.int64)
    truth = {0: [(np.arange(5, dtype=np.int64), {1: (v, np.ones(5, dtype=bool))})]}
    q = make_query([(1, cabi.TSKV_PT_I64)], ("count", "sum", "min", "max", "mean"))
    r = exact_aggregate(truth, q)
    S = 3 * I64_MAX + I64_MIN + 5
    assert r.exact_sums[1][0] == (S, 5)
    assert r.values[1][0] == S % 2**64
    assert r.values[4].view(np.float64)[0] == float(S) / 5.0
    assert r.values[2].view(np.int64)[0] == I64_MIN and r.values[3].view(np.int64)[0] == I64_MAX


def _check_case_against_oracle(case):
    name, step, w, origin, t0, n, kinds = case
    arena, descs, truth = geometry_arena(len(name), t0, step, n)
    for kind in kinds:
        ranges = geometry_ranges(kind, t0, step, n, w, origin)
        variants = [ranges] + ([split_ranges(ranges)] if len(ranges) == 1 else [])
        for qname, q in geometry_queries(case, ranges, truth):
            for rs in variants:
                q.time_ranges = rs
                what = "%s %s %s %s" % (name, kind, qname, rs)
                try:
                    exp = exact_aggregate(truth, q)
                except ReferenceError as e:
                    if e.status == cabi.TSKV_ERR_UNSUPPORTED:  # (the oracle has no key budget)
                        assert sel_unsupported(q, truth), what
                        continue
                    with pytest.raises(orc.OracleError) as oe:
                        orc.scan_aggregate(arena, descs, q)
                    assert oe.value.status == e.status, what
                    continue
                got = orc.scan_aggregate(arena, descs, q)
                # FIRST / LAST where a page's timestamps are distinct (with step 0 every row ties)
                assert_matches_exact(got, exp, what=what, int_mean=False,
                                     first_last=bool(step) and not raw_key_edge(q, truth))


@pytest.mark.parametrize("case", GEOMETRY_CASES, ids=[c[0] for c in GEOMETRY_CASES])
def test_reference_matches_oracle_on_the_geometry_sweep(case):
    _check_case_against_oracle(case)


def test_bucket_grid_one_short_is_an_error_for_both():
    for case in (c for c in GEOMETRY_CASES if c[5] >= 31 and c[2] < 2**40):
        name, step, w, origin, t0, n, _ = case
        arena, descs, truth = geometry_arena(len(name), t0, step, n)
        q = geometry_queries(case, [], truth)[0][1]
        if q.n_buckets < 2:
            continue
        for fbs, nb in ((q.first_bucket_start + w, q.n_buckets - 1), (q.first_bucket_start, q.n_buckets - 1)):
            q.first_bucket_start, q.n_buckets = fbs, nb
            with pytest.raises(ReferenceError):
                exact_aggregate(truth, q)
            with pytest.raises(orc.OracleError) as oe:
                orc.scan_aggregate(arena, descs, q)
            assert oe.value.status == cabi.TSKV_ERR_BUCKET_RANGE
        break


def test_f64_sum_classes():
    """NaN and infinities decide an f64 sum in every order; a finite one is exactly rounded, +0.0 when zero; a sum that
    overflows in some orders only is refused."""
    inf, nan, big = math.inf, math.nan, DBL_MAX
    assert math.isnan(f64_sum_class([1.0, nan])[0]) and math.isnan(f64_sum_class([inf, -inf, 2.0])[0])
    assert f64_sum_class([-inf, 5.0, -big]) == (-inf, 0.0)
    assert f64_sum_class([big, big, -1.0]) == (inf, 0.0)            # every order overflows: exact sum >= 2 DBL_MAX
    assert f64_sum_class([-big] * 3) == (-inf, 0.0)
    assert f64_sum_class([big]) == (big, big) and f64_sum_class([-big, -0.0]) == (-big, big)
    s = f64_sum_class([-0.0, -0.0])[0]
    assert s == 0 and math.copysign(1, s) == 1
    assert f64_sum_class([1e300, -1e300, 5e-324]) == (5e-324, 2e300)
    for x in ([big, -big, 1.0], [inf, -big, -big], [big, big, -big, -big]):
        with pytest.raises(OrderDependentSum):
            f64_sum_class(x)


@pytest.mark.parametrize("n", F64_LENGTHS)
def test_reference_matches_oracle_on_f64_edges(n):
    """The extended reference against the oracle on the f64 edge arenas: COUNT / MIN / MAX bit for bit, SUM / MEAN by
    class and within the bound (the oracle sums in row order, from +0.0)."""
    arena, descs, truth = f64_edge_arena(n, n)
    for name, q, extra in f64_edge_queries(n):
        exp = f64_edge_expected(truth, q, extra)
        if "group_ids" in extra or "slide" in extra:
            continue  # (the oracle has no GROUP BY tags or sliding windows; their references build on this one)
        got = orc.scan_aggregate(arena, descs, q)
        assert_matches_exact(got, exp, what="n=%d %s" % (n, name))
        # the arenas reach every class
        if name == "by_series" and n >= 31:
            c = exp.center[1]
            assert np.isnan(c).any() and np.isposinf(c).any() and np.isneginf(c).any() and np.isfinite(c).any()


# ---- FIRST / LAST, tombstones and the overlap merge --------------------------------------------------------------------
# The reference's FIRST / LAST, tombstones and merge (tests/helpers.py) against the oracle on every arena of
# tests/exact_arenas.py: everything bit for bit but f64 SUM / MEAN (within the bound) and the integer MEAN.

def _against_oracle(arena, descs, truth, queries, tombstones=None, files=None, what=""):
    for name, q, extra in queries:
        if "group_ids" in extra or "slide" in extra:
            continue  # (the oracle has no GROUP BY tags or sliding windows)
        wh = "%s %s" % (what, name)
        try:
            exp = ea.expected(truth, q, extra, tombstones=tombstones, files=files)
        except ReferenceError as e:
            assert e.status == cabi.TSKV_ERR_UNSUPPORTED and sel_unsupported(q, truth), wh
            continue
        got = orc.scan_aggregate(arena, descs, q, tombstones=tombstones, chunk_files=files)
        assert_matches_exact(got, exp, what=wh, int_mean=False, first_last=not raw_key_edge(q, truth))


@pytest.mark.parametrize("kind", ea.FL_KINDS)
def test_reference_matches_oracle_on_first_last_arenas(kind):
    arena, descs, truth = ea.first_last_arena(kind)
    if kind == "raw":  # the time pages really are raw
        tp = descs[descs["phys_type"] == cabi.TSKV_PT_TIME]
        assert all(arena[int(d["offset"]) + 16 + (int(d["num_values"]) + 7) // 8] == cabi.TSKV_ENC_NULL for d in tp)
    _against_oracle(arena, descs, truth, ea.first_last_queries(truth), what=kind)


@pytest.mark.parametrize("width,bits", ea.BUDGET_WIDTHS)
def test_key_budget_edges(width, bits):
    """bits(2 width) + slot_bits = 61 and 62 are accepted (rows at both ends of rel), 63 is refused."""
    arena, descs, truth = ea.key_budget_arena(width)
    (name, q, _), = ea.key_budget_queries(width)
    if bits > 62:
        with pytest.raises(ReferenceError) as e:
            exact_aggregate(truth, q)
        assert e.value.status == cabi.TSKV_ERR_UNSUPPORTED
        return
    exp = exact_aggregate(truth, q)
    assert_matches_exact(orc.scan_aggregate(arena, descs, q), exp, what="width %d" % width)
    # at every time one slot holds no value: FIRST / LAST pick the lower of the other two
    assert exp.values[1].view(np.int64).tolist() == [1, 31] and exp.values[2].view(np.int64).tolist() == [20, 50]
    for span, bits in ((2**60 - 1, 62), (2**60, 63)):
        arena, descs, truth = ea.key_budget_arena(None, span)
        (name, q, _), = ea.key_budget_queries(None, unbucketed=True)
        if bits > 62:
            with pytest.raises(ReferenceError):
                exact_aggregate(truth, q)
        else:
            assert_matches_exact(orc.scan_aggregate(arena, descs, q), exact_aggregate(truth, q), what="span %d" % span)


@pytest.mark.parametrize("step,kind", ea.TB_CASES)
def test_reference_matches_oracle_with_tombstones(step, kind):
    arena, descs, truth = ea.tombstone_arena(step, kind)
    tombs = ea.tombstone_list(truth, step)
    _against_oracle(arena, descs, truth, ea.tombstone_queries(truth, step), tombstones=tombs, what="step %d %s" % (step, kind))


def test_reference_matches_oracle_on_the_merge_arena():
    arena, descs, truth, files = ea.merge_arena()
    queries = ea.merge_queries(truth)
    _against_oracle(arena, descs, truth, queries, files=files, what="merge")
    _against_oracle(arena, descs, truth, queries, files=files, tombstones=ea.merge_tombstones(truth), what="merge+tombs")
    # the sliding reference over the merged rows: its one-window-per-row case is the tumbling scan
    q, extra = ea.merge_sliding_query()
    ea.expected(truth, q, extra, files=files)
    q1 = make_query(ea.MG_FIELDS, ("count", "sum", "min", "max"), series_ids=q.series_ids, width=ea.MG_W,
                    origin=ea.MG_ORIGIN, first_bucket_start=q.first_bucket_start, n_buckets=q.n_buckets,
                    time_ranges=q.time_ranges)
    a, b = ea.expected(truth, q1, {"slide": ea.MG_W}, files=files), exact_aggregate(truth, q1, files=files)
    assert (a.values == b.values).all() and (a.validity == b.validity).all()


# ---- hand-worked cases -------------------------------------------------------------------------------------------------

def _one_col(truth, aggs=("count", "sum", "first", "last"), **kw):
    return make_query([(1, cabi.TSKV_PT_I64)], aggs, **kw)


def _col(truth_list):
    """{sid: [(ts, values with None for NULL)]} -> truth."""
    out = {}
    for sid, cgs in truth_list.items():
        for ts, vals in cgs:
            v = np.array([0 if x is None else x for x in vals], dtype=np.int64)
            out.setdefault(sid, []).append((np.array(ts, dtype=np.int64), {1: (v, np.array([x is not None for x in vals]))}))
    return out


def _cells(r, agg):
    j = r.names.index((1, agg))
    return [int(v) if ok else None for v, ok in zip(r.values[j].view(np.int64), r.validity[j])]


def _arena(truth):
    b = datagen.ArenaBuilder()
    for sid, cgs in truth.items():
        for ts, cols in cgs:
            v, ok = cols[1]
            b.add_column_group(sid, ts, [(1, cabi.TSKV_PT_I64, v, ok)])
    return b.finish()


def _both(truth, q, **kw):
    """The reference, checked against the oracle."""
    exp = exact_aggregate(truth, q, tombstones=kw.get("tombstones"), files=kw.get("files"))
    arena, descs = _arena(truth)
    assert_matches_exact(orc.scan_aggregate(arena, descs, q, tombstones=kw.get("tombstones"), chunk_files=kw.get("files")),
                         exp, int_mean=False)
    return exp


def test_null_first_row_drops_the_run():
    """Series 0's run in bucket [10, 20) starts with a NULL at t=10: it contributes no FIRST, though its t=12 row holds
    a value; series 1's later value at t=15 is the FIRST. LAST: series 0's t=19 row is NULL, so series 1's t=18."""
    truth = _col({0: [([10, 12, 19], [None, 5, None])], 1: [([15, 18], [7, 8])]})
    r = _both(truth, _one_col(truth, width=10, first_bucket_start=10, n_buckets=1))
    assert _cells(r, "first") == [7] and _cells(r, "last") == [8] and _cells(r, "count") == [3]
    # by series: series 0 has no FIRST / LAST at all
    r = _both(truth, _one_col(truth, width=10, first_bucket_start=10, n_buckets=1, group_by_series=True))
    assert _cells(r, "first") == [None, 7] and _cells(r, "last") == [None, 8]


def test_equal_time_tie_across_three_slots():
    """Three slots hold rows at t=5 and t=9: FIRST and LAST both take the lowest slot that has a value there - by
    selection order, not by series id."""
    truth = _col({3: [([5, 9], [30, 31])], 1: [([5, 9], [10, 11])], 2: [([5, 9], [None, 21])]})
    q = _one_col(truth, series_ids=np.array([2, 3, 1], dtype=np.uint32), width=10, first_bucket_start=0, n_buckets=1)
    r = exact_aggregate(truth, q)
    assert _cells(r, "first") == [30] and _cells(r, "last") == [21]
    q = _one_col(truth, series_ids=np.array([1, 2, 3], dtype=np.uint32), width=10, first_bucket_start=0, n_buckets=1)
    r = _both(truth, q)
    assert _cells(r, "first") == [10] and _cells(r, "last") == [11]


def test_tombstones_starting_and_ending_on_rows():
    truth = _col({0: [([10, 11, 12, 13, 14, 15], [1, 2, 3, 4, 5, 6])]})
    q = _one_col(truth, aggs=("count", "sum", "first", "last"))
    cases = [([(0, None, 11, 13)], 3, 1 + 5 + 6, 1, 6),          # rows 11-13 dropped
             ([(0, None, 10, 10), (0, None, 15, 15)], 4, 14, 2, 5),
             ([(0, 1, 10, 10)], 5, 20, None, 6),                  # the first value masked: the run has no FIRST
             ([(0, 1, 15, 16)], 5, 15, 1, None),
             ([(None, None, 9, 10), (0, 1, 14, 13)], 5, 20, 2, 6),  # global; an empty range
             ([(0, None, 16, 20), (1, None, 10, 15), (0, 2, 10, 15)], 6, 21, 1, 6)]  # past the rows; other keys
    for tb, count, s, first, last in cases:
        r = _both(truth, q, tombstones=cabi.tombstones(tb))
        assert (_cells(r, "count"), _cells(r, "sum"), _cells(r, "first"), _cells(r, "last")) == ([count], [s], [first], [last]), tb


def _merge_case(streams, aggs=("count", "sum", "first", "last")):
    """streams: [(file id, ts, values)] of series 7 -> the reference over buckets [1, 2) and [2, 3), checked against the
    oracle."""
    truth = _col({7: [(ts, v) for _, ts, v in streams]})
    files = np.array([f for f, _, _ in streams], dtype=np.uint64)
    return _both(truth, _one_col(truth, aggs, width=1, first_bucket_start=1, n_buckets=2), files=files)


def test_sort_merge_tables():
    """reader/sort_merge.rs:449-539 (the three tables the oracle is pinned to in tests/test_oracle_merge.py)."""
    r = _merge_case([(1, [1, 1, 1], [1, 2, 3]), (2, [1, 1, 2], [4, 5, 6]), (3, [1, 2, 2], [7, 8, 9])])
    assert _cells(r, "sum") == [7, 9] and _cells(r, "count") == [1, 1]
    r = _merge_case([(1, [1, 1, 1], [1, None, 3]), (2, [1, 1, 2], [None, 5, None]), (3, [1, 2, 2], [None, 8, None])])
    assert _cells(r, "sum") == [5, 8] and _cells(r, "first") == [5, 8] and _cells(r, "last") == [5, 8]
    r = _merge_case([(1, [1, 1, 1], [None] * 3), (2, [1, 1, 2], [None] * 3), (3, [1, 2, 2], [10, 20, 30])])
    assert _cells(r, "count") == [1, 1] and _cells(r, "sum") == [10, 30]


def test_touching_chunks_merge_and_separated_ones_do_not():
    """File 2 holds t = 10, 20 (NULL at 20); file 1 starts at 20 (touching: one group, the merged row at 20 takes file
    1's 5 since file 2's value is NULL) or at 21 (a gap of 1: two groups, plain rules). Bucket [20, 30): FIRST is 5
    merged; apart, file 2's run starts with a NULL and drops out, file 1's run starts at 21 with 6."""
    q = lambda truth: _one_col(truth, aggs=("count", "sum", "first", "last"), width=10, first_bucket_start=10, n_buckets=2)  # noqa: E731
    touch = _col({0: [([10, 20], [1, None]), ([20, 21, 25], [5, 6, 7])]})
    apart = _col({0: [([10, 20], [1, None]), ([21, 22, 25], [6, 8, 7])]})
    files = np.array([2, 1], dtype=np.uint64)
    r = exact_aggregate(touch, q(touch), files=files)
    assert _cells(r, "first") == [1, 5] and _cells(r, "count") == [1, 3] and _cells(r, "last") == [1, 7]
    r2 = exact_aggregate(apart, q(apart), files=files)
    assert _cells(r2, "first") == [1, 6] and _cells(r2, "count") == [1, 3] and _cells(r2, "last") == [1, 7]
    for truth, exp in ((touch, r), (apart, r2)):
        arena, descs = _arena(truth)
        assert_matches_exact(orc.scan_aggregate(arena, descs, q(truth), chunk_files=files), exp, int_mean=False)
    # the newer file wins a merged row; duplicates inside one chunk collapse, the chunk's later row winning
    dup = _col({0: [([20, 20, 20], [1, 2, None]), ([20], [None])]})
    r = exact_aggregate(dup, q(dup), files=np.array([3, 1], dtype=np.uint64))
    assert _cells(r, "count") == [0, 1] and _cells(r, "sum") == [None, 2]
