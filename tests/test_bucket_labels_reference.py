"""The exact reference with labelled time buckets, on hand-worked cases (no GPU): a row's output bucket is the label of
the edge bucket that holds it, several edge buckets fold into one cell, an output bucket no edge bucket maps to reads
like an empty bucket, and FIRST / LAST are refused."""
import numpy as np
import pytest

from cnosdb_b200 import cabi
from cnosdb_b200.engine import calendar_parts
from tests.edges_reference import exact_aggregate_edges
from tests.helpers import ReferenceError, make_query
from tests.labels_reference import exact_aggregate_grouped_labels, exact_aggregate_labels, label_bucket_index

FIELDS = [(1, cabi.TSKV_PT_I64)]
AGGS = ("count", "sum", "min", "max", "mean")
HOUR = 3600 * 10**9


def _col(res, agg):
    j = res.names.index((1, agg))
    return res.values[j].view(np.float64 if agg == "mean" else np.int64).tolist(), res.validity[j].tolist()


def _series(ts, vals):
    """One column group: int64 times, i64 values with None = NULL."""
    v = np.array([0 if x is None else x for x in vals], dtype=np.int64)
    ok = np.array([x is not None for x in vals], dtype=bool)
    return [(np.asarray(ts, dtype=np.int64), {1: (v, ok)})]


def _query(n_out, aggs=AGGS, **kw):
    return make_query(FIELDS, aggs, n_buckets=n_out, **kw)


def test_label_bucket_index():
    e = np.array([-10, -3, 0, 7], dtype=np.int64)
    lab = np.array([1, 0, 1], dtype=np.uint32)
    idx, ok = label_bucket_index(np.array([-11, -10, -4, -3, -1, 0, 6, 7]), e, lab)
    assert idx.tolist()[1:7] == [1, 1, 0, 0, 1, 1]
    assert ok.tolist() == [False, True, True, True, True, True, True, False]


def test_row_on_an_edge_takes_the_next_label():
    e = np.array([-5, 0, 10], dtype=np.int64)
    truth = {0: _series([-5, -1, 0, 9], [1, 2, 3, 4])}
    r = exact_aggregate_labels(truth, _query(2), e, [1, 0])
    assert _col(r, "count") == ([2, 2], [True, True])
    assert _col(r, "sum") == ([7, 3], [True, True])
    assert _col(r, "min") == ([3, 1], [True, True]) and _col(r, "max") == ([4, 2], [True, True])


def test_rows_outside_the_edges():
    e = np.array([-5, 0, 10], dtype=np.int64)
    for t in (-6, 10):  # one before edges[0], and edges[n] itself
        with pytest.raises(ReferenceError) as err:
            exact_aggregate_labels({0: _series([t, 1], [1, 2])}, _query(1), e, [0, 0])
        assert err.value.status == cabi.TSKV_ERR_BUCKET_RANGE
    # ... unless the time ranges leave them out
    r = exact_aggregate_labels({0: _series([-6, 1], [1, 2])}, _query(1, time_ranges=[(-5, 9)]), e, [0, 0])
    assert _col(r, "count") == ([1], [True])


def test_two_periods_of_one_page_fold_into_one_cell():
    """One column group over three hours: hour-of-day labels 5, 6, 5 over [05:00, 08:00) would be 3 periods; with the
    labels of two days' 05:00 hours equal, both periods land in cell 5 and their rows add up."""
    day = 24 * HOUR
    e = np.array([5 * HOUR, 6 * HOUR, 7 * HOUR, day + 5 * HOUR, day + 6 * HOUR], dtype=np.int64)
    lab = [5, 6, 7, 5]  # (the gap [07:00, day + 05:00) is edge bucket 2, labelled 7)
    ts = [5 * HOUR + 1, 5 * HOUR + 2, 6 * HOUR, day + 5 * HOUR, day + 6 * HOUR - 1]
    truth = {0: _series(ts, [10, None, 20, 30, -4])}
    r = exact_aggregate_labels(truth, _query(24), e, lab)
    count, ok = _col(r, "count")
    assert count[5] == 3 and count[6] == 1 and sum(count) == 4
    assert _col(r, "sum")[0][5] == 36 and _col(r, "min")[0][5] == -4 and _col(r, "max")[0][5] == 30
    assert _col(r, "mean")[0][5] == 12.0


def test_output_bucket_without_edge_bucket_is_empty():
    e = np.array([0, 10, 20], dtype=np.int64)
    truth = {0: _series([1, 15], [3, 4])}
    r = exact_aggregate_labels(truth, _query(4), e, [3, 1])
    assert _col(r, "count") == ([0, 1, 0, 1], [True] * 4)
    assert _col(r, "sum") == ([0, 4, 0, 3], [False, True, False, True])
    assert _col(r, "min")[1] == [False, True, False, True]


def test_identity_labels_equal_the_edge_reference():
    e = np.array([0, 7, 19, 40, 41, 100], dtype=np.int64)
    rng = np.random.default_rng(3)
    truth = {s: _series(np.sort(rng.choice(100, 30, replace=False)), rng.integers(-50, 50, 30).tolist()) for s in range(5)}
    q = _query(len(e) - 1)
    a = exact_aggregate_labels(truth, q, e, np.arange(len(e) - 1))
    b = exact_aggregate_edges(truth, q, e)
    assert (a.values == b.values).all() and (a.validity == b.validity).all()


def test_hour_of_day_equals_folded_hours():
    """calendar_parts('hour') over three days == the 72 hourly buckets of the edge reference folded by hour of day."""
    e, lab, values = calendar_parts("hour", 0, 3 * 24 * HOUR - 1)
    rng = np.random.default_rng(8)
    truth = {s: _series(np.sort(rng.choice(3 * 24 * HOUR, 200, replace=False)), rng.integers(-99, 99, 200).tolist())
             for s in range(3)}
    agg = ("count", "sum")
    r = exact_aggregate_labels(truth, _query(24, agg), e, lab)
    fine = exact_aggregate_edges(truth, _query(72, agg), e)
    for name in agg:
        v, _ = _col(fine, name)
        assert _col(r, name)[0] == np.array(v).reshape(3, 24).sum(axis=0).tolist()
    assert values.tolist() == list(range(24))


def test_grouped_labels():
    e = np.array([0, 10, 20, 30], dtype=np.int64)
    truth = {5: _series([1, 11, 21], [1, 2, 3]), 9: _series([2, 12, 22], [10, 20, 30])}
    g = exact_aggregate_grouped_labels(truth, _query(2), [1, 0], 2, e, [0, 1, 0])
    assert _col(g, "sum") == ([40, 20, 4, 2], [True] * 4)  # group 0 = series 9, group 1 = series 5
    r = exact_aggregate_labels(truth, _query(2, group_by_series=True), e, [0, 1, 0])
    assert _col(r, "sum") == ([4, 2, 40, 20], [True] * 4)


@pytest.mark.parametrize("agg", ["first", "last"])
def test_first_last_are_refused(agg):
    e = np.array([0, 10], dtype=np.int64)
    with pytest.raises(ReferenceError) as err:
        exact_aggregate_labels({0: _series([1], [1])}, _query(1, ("count", agg)), e, [0])
    assert err.value.status == cabi.TSKV_ERR_UNSUPPORTED
