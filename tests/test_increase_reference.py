"""The exact increase reference (tests/increase_reference.py) against the reference's increase.slt answers and hand
cases: resets, equal runs, one value, NULLs, i64 / u64 wrapping at the extremes, NaN / +-inf / +-0.0 under totalOrder,
time order against row order, and buckets; and the vectorized reference of the scale test against the exact one."""
import math

import numpy as np

from cnosdb_b200 import cabi
from cnosdb_b200.engine import PushedAggregate, QueryOption
from tests.covariance_reference import TB2_TYPES
from tests.helpers import bucket_index
from tests.increase_reference import exact_increase_cells, increase_bits, increase_cells_np, load_golden

I64, U64, F64 = cabi.TSKV_PT_I64, cabi.TSKV_PT_U64, cabi.TSKV_PT_F64
PT = {"u64": U64, "i64": I64, "f64": F64}
DT = {I64: np.int64, U64: np.uint64, F64: np.float64}


def typed(bits, pt):
    return np.uint64(bits).view(DT[pt]).item()


def one_series(ts, vals, pt, valid=None, width=0, n_buckets=1, fbs=0):
    ts = np.asarray(ts, dtype=np.int64)
    v = np.asarray(vals, dtype=DT[pt])
    ok = np.ones(len(v), dtype=bool) if valid is None else np.asarray(valid, dtype=bool)
    truth = {0: [(ts, {1: (v, ok)})]}
    q = QueryOption([PushedAggregate(1, pt, ["increase"])], first_bucket_start=fbs, n_buckets=n_buckets, width=width)
    return exact_increase_cells(truth, q, 1, pt, n_buckets)


def golden_tb2(g, name):
    t = g["tables"]["func_tb2"]
    cols = t["columns"]
    ts = np.array([int(r[0]) for r in t["rows"]], dtype=np.int64)
    kind = TB2_TYPES[name]
    vals = [r[cols.index(name)] for r in t["rows"]]
    v = np.array([float(x) for x in vals]) if kind == "f64" else np.array([int(x) for x in vals], dtype=DT[PT[kind]])
    return ts, v, PT[kind]


def test_golden_func_tb2():
    g = load_golden()
    assert {a["column"] for a in g["func_tb2"]} == {"f0", "f1", "f4"}
    for a in g["func_tb2"]:
        ts, v, pt = golden_tb2(g, a["column"])
        r, ok, _ = one_series(ts, v, pt)
        assert ok[0] and repr(typed(r[0], pt)) == a["expected"], (a, typed(r[0], pt))


def test_golden_test_increase_grouped():
    g = load_golden()["test_increase"]
    assert len(g["series"]) == 2
    for s in g["series"]:
        rows = s["rows"]
        ts = np.array([np.datetime64(r["time"].replace(" ", "T"), "ns").astype(np.int64) for r in rows])
        r, ok, _ = one_series(ts, [r["f0"] for r in rows], I64)
        assert ok[0] and typed(r[0], I64) == g["group_by_t0"]["expected"][rows[0]["t0"]]


def test_golden_refused_types():
    assert {(r["column"], r["type"]) for r in load_golden()["refused"]} == {("f2", "Boolean"), ("f3", "Utf8")}


def test_resets_equal_runs_one_value_nulls():
    assert increase_bits([5], I64) == (0, 0.0)
    assert increase_bits([], I64) == (None, 0.0)
    assert increase_bits([3, 3, 3], U64)[0] == 0
    assert increase_bits([1, 4, 4, 2, 7, 1], I64)[0] == 3 + 2 + 5 + 1
    # NULL operand values are left out: the pair spans them
    r, ok, _ = one_series([1, 2, 3, 4], [10, 0, 0, 12], I64, valid=[1, 0, 0, 1])
    assert ok[0] and typed(r[0], I64) == 2
    r, ok, _ = one_series([1, 2], [10, 12], I64, valid=[0, 0])
    assert not ok[0]


def test_time_order_not_row_order():
    r, _, _ = one_series([30, 10, 20], [3, 1, 2], U64)
    assert typed(r[0], U64) == 2
    r, _, _ = one_series([10, 20, 30], [3, 1, 2], U64)
    assert typed(r[0], U64) == 2  # (reset to 1, then +1)


def test_buckets_do_not_pair_across():
    r, ok, _ = one_series([0, 5, 10, 15], [1, 2, 10, 11], I64, width=10, n_buckets=2)
    assert ok.all() and [typed(x, I64) for x in r] == [1, 1]


def test_integer_wrap():
    big = 2**63 - 1
    assert typed(increase_bits([-2**63, big], I64)[0], I64) == -1  # big - MIN wraps to -1
    assert typed(increase_bits([0, big, 0, big], I64)[0], I64) == -2  # big + 0 + big wraps
    assert typed(increase_bits([big, -2**63], I64)[0], I64) == -2**63  # a reset adds the (negative) value
    assert increase_bits([0, 2**64 - 1, 0, 2**64 - 1], U64)[0] == 2**64 - 2
    assert increase_bits([2**63, 1], U64)[0] == 1  # unsigned compare: 1 < 2^63 is a reset


def test_f64_special_values():
    f = lambda vals: typed(increase_bits(vals, F64)[0], F64)
    assert f([1.0, 2.5, 0.5, 4.0]) == 1.5 + 0.5 + 3.5
    assert math.isnan(f([1.0, math.nan]))  # +NaN is above every number: adds NaN - 1
    assert f([math.nan, 1.0]) == 1.0  # a number after +NaN is a reset
    neg_nan = float(np.uint64(0xFFF8000000000000).view(np.float64))
    assert math.isnan(f([neg_nan, 1.0]))  # -NaN is below every number: 1.0 adds 1.0 - NaN
    assert math.isnan(f([1.0, neg_nan]))  # a reset adds the NaN itself
    assert f([1.0, math.inf]) == math.inf
    assert f([math.inf, 1.0]) == 1.0
    assert f([-math.inf, 1.0]) == math.inf
    assert np.float64(f([0.0, -0.0])).view(np.uint64) == np.float64(0.0).view(np.uint64)  # -0.0 < +0.0: a reset adds -0.0
    assert f([-0.0, 0.0]) == 0.0
    assert f([2.0, 2.0]) == 0.0


def flat_rows(truth, col, pt, nb, bucket):
    """(cells, times, bit patterns) of every valid row of `col`, cell = series slot * nb + bucket(times) (rows without a
    bucket, bucket < 0, left out): the vectorized reference's input."""
    cells, times, bits = [], [], []
    for slot, sid in enumerate(sorted(truth)):
        for ts, cols in truth[sid]:
            if col not in cols:
                continue
            v, ok = cols[col]
            b = bucket(np.asarray(ts, dtype=np.int64))
            keep = np.asarray(ok, dtype=bool) & (b >= 0)
            cells.append(slot * nb + b[keep])
            times.append(np.asarray(ts, dtype=np.int64)[keep])
            bits.append(np.asarray(v, dtype=DT[pt])[keep].view(np.uint64))
    return np.concatenate(cells), np.concatenate(times), np.concatenate(bits)


def random_truth(rng, pt, n_series=6):
    """Series of 1-4 column groups, written out of time order, with NULLs, counter resets, runs of equal values and
    (integers) values near the type's extremes that wrap the sum; f64 with NaN, +-inf and +-0.0."""
    truth = {}
    for sid in range(n_series):
        cgs, t = [], int(rng.integers(-10**6, 10**6))
        for _ in range(int(rng.integers(1, 5))):
            n = int(rng.integers(1, 60))
            ts = t + np.cumsum(rng.integers(1, 1000, n)).astype(np.int64)
            t = int(ts[-1]) + 1
            walk = np.cumsum(rng.integers(-3, 6, n))
            walk[rng.random(n) < 0.1] = 0  # resets
            if pt == F64:
                v = walk.astype(np.float64) + np.round(rng.random(n), 2)
                sp = rng.random(n) < 0.05
                v[sp] = rng.choice([np.nan, np.inf, -np.inf, 0.0, -0.0], int(sp.sum()))
            elif pt == I64:
                v = walk.astype(np.int64) + (0, 2**63 - 50, -2**63 + 50)[int(rng.integers(0, 3))]
            else:
                v = walk.astype(np.int64).view(np.uint64) + np.uint64((0, 2**64 - 50, 2**63)[int(rng.integers(0, 3))])
            cgs.append((ts, {1: (v, rng.random(n) > 0.2)}))
        truth[sid] = [cgs[k] for k in rng.permutation(len(cgs))]
    return truth


def test_vectorized_reference_matches_the_exact_one():
    """increase_cells_np (the reference of the scale test) equals exact_increase_cells on random truths, GROUP BY series
    over tumbling buckets and over edges (rows outside the edges dropped): integers bit for bit, f64 bit for bit too
    (both add in time order per cell) and the same magnitudes."""
    rng = np.random.default_rng(77)
    for trial in range(24):
        pt = (I64, U64, F64)[trial % 3]
        truth = random_truth(rng, pt)
        lo = min(int(ts.min()) for cgs in truth.values() for ts, _ in cgs)
        hi = max(int(ts.max()) for cgs in truth.values() for ts, _ in cgs)
        if trial % 2:
            e = np.unique(np.concatenate([[lo + 5], rng.integers(lo, hi, 6), [hi - 5]])).astype(np.int64)
            q = QueryOption([PushedAggregate(1, pt, ["increase"])], n_buckets=e.size - 1, group_by_series=True)
            kw = dict(edges=e)
            bucket = lambda t: np.where((t >= e[0]) & (t < e[-1]), np.searchsorted(e, t, side="right") - 1, -1)  # noqa: E731
        else:
            w = int(rng.integers(500, 20000))
            fbs = lo - lo % w
            nb = (hi - fbs) // w + 1
            q = QueryOption([PushedAggregate(1, pt, ["increase"])], width=w, first_bucket_start=fbs, n_buckets=nb,
                            group_by_series=True)
            kw = {}
            bucket = lambda t: np.where(bucket_index(t, q)[1], bucket_index(t, q)[0], -1)  # noqa: E731
        nb = q.n_buckets
        n_cells = len(truth) * nb
        v_e, ok_e, mag_e = exact_increase_cells(truth, q, 1, pt, n_cells, **kw)
        v, ok, mag = increase_cells_np(*flat_rows(truth, 1, pt, nb, bucket), pt, n_cells)
        np.testing.assert_array_equal(ok, ok_e, err_msg=str(trial))
        np.testing.assert_array_equal(v[ok_e], v_e[ok_e], err_msg=str(trial))
        np.testing.assert_array_equal(mag[ok_e], mag_e[ok_e], err_msg=str(trial))
        assert ok_e.sum() >= 3, trial
