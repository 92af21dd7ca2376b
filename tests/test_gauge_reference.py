"""tests/gauge_reference.py against a literal restatement of the reference's update_batch + build over random batch
splits, its pane fold against row expansion, and engine.gauge_stat's NULL rules (no GPU)."""
import numpy as np

from cnosdb_b200 import cabi
from cnosdb_b200.engine import GAUGE_STATS, QueryOption, PushedAggregate, gauge_stat
from cnosdb_b200.engine import sliding_window_grid
from tests.gauge_reference import (gauge_of, golden_cases, golden_refused, pane_points, sliding_points,
                                   update_batch_reference)
from tests.helpers import random_arena
from tests.sliding_reference import expand_aggregate

I64, F64 = cabi.TSKV_PT_I64, cabi.TSKV_PT_F64


def test_positions_equal_update_batch_over_random_splits():
    """Points in random order, cut into random batches: the exact reference equals update_batch + build."""
    rng = np.random.default_rng(1)
    for _ in range(500):
        n = int(rng.integers(1, 40))
        t = rng.choice(10_000, n, replace=False).astype(int)
        pts = [(int(x), 0, int(rng.integers(0, 1 << 60))) for x in t]
        cuts = [0] + sorted(int(c) for c in rng.choice(np.arange(1, n + 1), int(rng.integers(0, n)), replace=False) if c < n) + [n]
        out, ok = gauge_of(sorted(pts))
        n_r, first, second, pen, last = update_batch_reference(pts, cuts)
        assert out[0] == n_r == n
        assert (out[1], out[3], out[5], out[7]) == (first[0], second[0], pen[0], last[0])
        assert (out[2], out[4], out[6], out[8]) == (first[2], second[2], pen[2], last[2])


def test_ties_give_the_same_timestamps():
    pts = [(5, 1, 10), (5, 0, 20), (7, 0, 30), (7, 2, 40)]
    out, _ = gauge_of(sorted(pts, key=lambda p: (p[0], p[1])))
    n, first, second, pen, last = update_batch_reference(pts, [0, 4])
    assert (out[1], out[3], out[5], out[7]) == (first[0], second[0], pen[0], last[0])
    assert out[2] == 20 and out[8] == 40  # the lower slot first


def test_one_and_two_points():
    assert gauge_of([(3, 0, 9)])[0] == [1, 3, 9, 3, 9, 3, 9, 3, 9]
    assert gauge_of([(3, 0, 9), (4, 0, 8)])[0] == [2, 3, 9, 4, 8, 3, 9, 4, 8]
    assert gauge_of([])[1] == [True] + [False] * 8


def test_pane_fold_equals_row_expansion():
    """The pane fold (the scan's construction) equals row expansion on divisible and non-divisible grids, and the
    expansion's points per window number the COUNT of tests/sliding_reference.py's Expand plan."""
    rng = np.random.default_rng(2)
    a, d, truth = random_arena(rng, n_series=6, n_points=120, fields=((1, I64), (2, F64)), null_frac=0.2, multi_cg=True)
    lo = min(int(ts[0]) for cgs in truth.values() for ts, _ in cgs if len(ts))
    hi = max(int(ts[-1]) for cgs in truth.values() for ts, _ in cgs if len(ts))
    for window, slide in ((40_000, 10_000), (30_000, 20_000), (10_000, 10_000), (50_000, 7_000)):
        for gbs in (False, True):
            fbs, n_b = sliding_window_grid(lo, hi, window, slide)
            q = QueryOption([PushedAggregate(1, I64, ["count"])], width=window, origin=0, first_bucket_start=fbs,
                            n_buckets=n_b, group_by_series=gbs)
            rows = sliding_points(truth, q, 1, I64, slide, 6)
            assert pane_points(truth, q, 1, I64, slide) == rows, (window, slide, gbs)
            exp = expand_aggregate(truth, q, slide)
            count = np.asarray(exp.values[exp.names.index((1, "count"))]).astype(np.int64)
            got = np.zeros(count.size, dtype=np.int64)
            for cell, pts in rows.items():
                got[cell] = len(pts)
            np.testing.assert_array_equal(got, count, err_msg="%d/%d gbs=%s" % (window, slide, gbs))


def test_gauge_stat_null_rules():
    n = np.array([0, 1, 2, 3], dtype=np.uint64)
    ft = np.array([0, 5, 5, -(2**63)], dtype=np.int64)
    lt = np.array([0, 5, 9, 2**63 - 1], dtype=np.int64)
    fv = np.array([0.0, 1.0, 1.0, 1.0])
    sv = np.array([0.0, 1.0, 4.0, 2.0])
    pv = np.array([0.0, 1.0, 1.0, 2.0])
    lv = np.array([0.0, 1.0, 4.0, 3.0])
    args = (n, ft, fv, ft, sv, ft, pv, lt, lv)
    v, ok = gauge_stat("delta", *args)
    assert ok.tolist() == [False, True, True, True] and v[2] == 3.0
    v, ok = gauge_stat("time_delta", *args)
    assert ok.tolist() == [False, True, True, False] and v[2] == 4
    v, ok = gauge_stat("rate", *args)
    assert ok.tolist() == [False, False, True, False] and v[2] == 0.75
    assert gauge_stat("idelta_left", *args)[0][2] == 3.0 and gauge_stat("idelta_right", *args)[0][3] == 1.0
    for name in GAUGE_STATS:
        assert not gauge_stat(name, *args)[1][0]


def test_golden_answers_from_the_reference():
    """The exact reference on the slt tables, through gauge_stat, gives every gauge_agg / accessor answer of
    gauge_slt.json (func_tb2.f0 is BIGINT UNSIGNED: coerced to f64)."""
    cases = golden_cases()
    assert len(cases) >= 40
    for case in cases:
        case.check(case.reference_outputs)
    assert golden_refused() == ["Boolean", "Timestamp", "Utf8"]
