"""The exact reference of tests/helpers.py checked on its own (no GPU): its window arithmetic against the reference's
known-answer vectors and the oracle's restatement, and its aggregates against the oracle on every arena of the bucket
geometry sweep. COUNT / SUM / MIN / MAX must agree bit for bit; f64 sums within the order-free bound; the integer MEAN is
not compared (the oracle keeps an f64 running sum, the reference the exact one)."""
import math

import numpy as np
import pytest

from oracle import pyoracle as orc
from tests.helpers import (DBL_MAX, F64_LENGTHS, GEOMETRY_CASES, I64_MAX, I64_MIN, OrderDependentSum, ReferenceError,
                           assert_matches_exact, ceil_sliding_window, exact_aggregate, f64_edge_arena, f64_edge_expected,
                           f64_edge_queries, f64_sum_class, floor_sliding_window, geometry_arena, geometry_queries,
                           geometry_ranges, make_query, sliding_window, split_ranges)
from cnosdb_b200 import cabi


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
                    with pytest.raises(orc.OracleError) as oe:
                        orc.scan_aggregate(arena, descs, q)
                    assert oe.value.status == e.status, what
                    continue
                got = orc.scan_aggregate(arena, descs, q)
                assert_matches_exact(got, exp, what=what, int_mean=False)


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
