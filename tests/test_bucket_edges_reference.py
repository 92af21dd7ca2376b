"""The exact reference with explicit time-bucket edges, on hand-worked cases (no GPU): a row's bucket is
the last edge at or before it, FIRST / LAST keep the (page, bucket) run semantics of the tumbling scan, and the key
budget comes from the longest bucket."""
import numpy as np
import pytest

from cnosdb_b200 import cabi
from cnosdb_b200.engine import calendar_edges
from tests.edges_reference import (edge_bucket_index, edge_rel_bits, exact_aggregate_edges,
                                   exact_aggregate_grouped_edges)
from tests.helpers import ReferenceError, make_query

FIELDS = [(1, cabi.TSKV_PT_I64)]
AGGS = ("count", "sum", "min", "max", "first", "last")
DAY = 86400 * 10**9


def _col(res, agg):
    j = res.names.index((1, agg))
    return res.values[j].view(np.int64).tolist(), res.validity[j].tolist()


def _series(ts, vals):
    """One column group: int64 times, i64 values with None = NULL."""
    v = np.array([0 if x is None else x for x in vals], dtype=np.int64)
    ok = np.array([x is not None for x in vals], dtype=bool)
    return [(np.asarray(ts, dtype=np.int64), {1: (v, ok)})]


def _query(edges, **kw):
    return make_query(FIELDS, AGGS, n_buckets=len(edges) - 1, **kw)


def test_bucket_index_floors_on_edges():
    e = np.array([-10, -3, 0, 7], dtype=np.int64)
    idx, ok = edge_bucket_index(np.array([-11, -10, -4, -3, -1, 0, 6, 7]), e)
    assert idx.tolist()[1:7] == [0, 0, 1, 1, 2, 2]
    assert ok.tolist() == [False, True, True, True, True, True, True, False]


def test_month_run_with_null_first_row_drops_first():
    """The (page, month) run whose first selected row is NULL contributes no FIRST (first.rs:91-94); its LAST and the
    other month are unaffected."""
    e = calendar_edges("month", -40 * DAY, -1)  # Nov 1969, Dec 1969
    assert len(e) == 3
    truth = {0: _series([e[0] + 5, e[0] + 9, e[1] + 1, e[1] + 2], [None, 11, 20, 21])}
    r = exact_aggregate_edges(truth, _query(e), e)
    assert _col(r, "count") == ([1, 2], [True, True])
    assert _col(r, "first") == ([0, 20], [False, True])
    assert _col(r, "last") == ([11, 21], [True, True])
    assert _col(r, "sum") == ([11, 41], [True, True])


def test_tie_across_series_at_the_same_time():
    """Two series with a row at the same time: FIRST and LAST both take the lower slot's value."""
    e = np.array([0, 100, 300], dtype=np.int64)
    truth = {5: _series([10, 150], [1, 3]), 9: _series([10, 150], [2, 4])}
    r = exact_aggregate_edges(truth, _query(e), e)
    assert _col(r, "first") == ([1, 3], [True, True])
    assert _col(r, "last") == ([1, 3], [True, True])
    assert _col(r, "min") == ([1, 3], [True, True]) and _col(r, "max") == ([2, 4], [True, True])
    g = exact_aggregate_grouped_edges(truth, _query(e), [1, 0], 2, e)  # each series its own group
    assert _col(g, "first") == ([2, 4, 1, 3], [True] * 4)


def test_row_on_an_edge_opens_the_next_bucket():
    e = np.array([-5, 0, 10], dtype=np.int64)
    truth = {0: _series([-5, -1, 0, 9], [1, 2, 3, 4])}
    r = exact_aggregate_edges(truth, _query(e), e)
    assert _col(r, "count") == ([2, 2], [True, True])
    assert _col(r, "first") == ([1, 3], [True, True]) and _col(r, "last") == ([2, 4], [True, True])


def test_rows_outside_the_edges():
    e = np.array([-5, 0, 10], dtype=np.int64)
    for t in (-6, 10):  # one before edges[0], and edges[n] itself
        with pytest.raises(ReferenceError) as err:
            exact_aggregate_edges({0: _series([t, 1], [1, 2])}, _query(e), e)
        assert err.value.status == cabi.TSKV_ERR_BUCKET_RANGE
    # ... unless the time ranges leave them out
    r = exact_aggregate_edges({0: _series([-6, 1], [1, 2])}, _query(e, time_ranges=[(-5, 9)]), e)
    assert _col(r, "count") == ([0, 1], [True, True])


def test_key_budget_is_the_longest_bucket():
    """Yearly buckets at ns precision: rel needs 55 bits, 7 slot bits remain - FIRST / LAST across up to 128 series."""
    e = calendar_edges("year", 0, 3 * 365 * DAY)  # 1970 .. 1973 (1972 is a leap year)
    assert edge_rel_bits(e) == 55
    assert 7 + 55 <= 62
    ts = [int(e[0]) + 1]

    def truth(n):
        return {s: _series(ts, [s]) for s in range(n)}
    r = exact_aggregate_edges(truth(128), _query(e), e)
    assert _col(r, "first")[0][0] == 0
    with pytest.raises(ReferenceError) as err:
        exact_aggregate_edges(truth(129), _query(e), e)
    assert err.value.status == cabi.TSKV_ERR_UNSUPPORTED
    # GROUP BY series needs no slot bits
    r = exact_aggregate_edges(truth(129), _query(e, group_by_series=True), e)
    assert r.values.shape[1] == 129 * (len(e) - 1)
