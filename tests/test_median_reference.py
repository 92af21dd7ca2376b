"""tests/median_reference.py on its own (CPU): the reference's three median answers of approx_median.slt
(tests/golden/median_slt.json) and hand-worked cases of the even-n rule, the type orders and the row selection."""
import json
import math
import os

import numpy as np

from cnosdb_b200 import cabi
from cnosdb_b200.engine import PushedAggregate, QueryOption
from tests.median_reference import exact_median_cells, median_bits, selected_values

I64, U64, F64 = cabi.TSKV_PT_I64, cabi.TSKV_PT_U64, cabi.TSKV_PT_F64
GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "median_slt.json")
TYPES = {"bigint": I64, "bigint unsigned": U64, "double": F64}
M64 = (1 << 64) - 1


def load_golden():
    with open(GOLDEN) as f:
        return json.load(f)


def golden_column(g, name):
    """(typed values, valid) of one column of test_approx_median_tbl in row order."""
    t = g["table"]
    pt = TYPES[t["types"][name]]
    raw = [r[t["columns"].index(name)] for r in t["rows"]]
    ok = np.array([v != "NULL" for v in raw])
    if pt == F64:
        return pt, np.array([float(v) if v != "NULL" else 0.0 for v in raw]), ok
    return pt, np.array([int(v) if v != "NULL" else 0 for v in raw], dtype=np.int64 if pt == I64 else np.uint64), ok


def f(bits):
    return float(np.uint64(bits).view(np.float64))


def fb(x):
    return int(np.float64(x).view(np.uint64))


def test_golden_answers():
    g = load_golden()
    assert [c["column"] for c in g["checks"]] == ["d_val", "val", "u_val"]
    for c in g["checks"]:
        pt, v, ok = golden_column(g, c["column"])
        m = median_bits(list(v[ok]), pt)
        if pt == F64:
            assert repr(f(m)) == c["expected"], (c, f(m))
        elif pt == I64:
            assert m == int(c["expected"]) & M64
        else:
            assert m == int(c["expected"])


def test_integer_even_rule():
    assert median_bits([-3, 0], I64) == (-1) & M64          # (-3 + 0) / 2 truncates toward zero
    assert median_bits([-4, -1], I64) == (-2) & M64
    assert median_bits([-5, 0], I64) == (-2) & M64
    mx = np.iinfo(np.int64).max
    assert median_bits([mx, mx], I64) == (-1) & M64         # MAX + MAX wraps to -2
    mn = np.iinfo(np.int64).min
    assert median_bits([mn, mn], I64) == 0                  # MIN + MIN wraps to 0
    assert median_bits([mn, mx], I64) == 0                  # -1 / 2 truncates to 0
    assert median_bits([2**64 - 1, 3], U64) == 1            # wrapping add: 2 / 2
    assert median_bits([2**64 - 2, 2**64 - 2], U64) == (2**64 - 4) // 2
    assert median_bits([7, 1, 5], I64) == 5 and median_bits([7, 1, 5, 9], U64) == 6
    assert median_bits([2**63, 0, 2**63 + 2, 1], U64) == (1 + 2**63) // 2  # u64 order, not i64's


def test_f64_special_values():
    nan = float("nan")
    assert f(median_bits([1.0, 2.0, 3.0], F64)) == 2.0
    assert f(median_bits([1.0, 4.0], F64)) == 2.5
    assert median_bits([1.0, nan], F64) == fb(nan) | 0x0008000000000000       # NaN sorts above +inf
    assert median_bits([1.0, 2.0, nan], F64) == fb(2.0)
    neg_nan = 0xFFF8000000000001
    assert median_bits([f(neg_nan), 1.0], F64) == neg_nan                        # -NaN sorts below -inf: lo
    assert median_bits([float("-inf"), float("inf")], F64) == 0xFFF8000000000000
    assert median_bits([float("-inf"), 5.0, float("inf")], F64) == fb(5.0)
    assert median_bits([float("inf"), float("inf")], F64) == fb(float("inf"))
    assert median_bits([-0.0, 0.0], F64) == fb(0.0)                              # -0.0 < +0.0, (-0.0 + 0.0) / 2
    assert median_bits([0.0, -0.0, -0.0], F64) == fb(-0.0)
    assert median_bits([1e308, 1e308], F64) == fb(float("inf"))                  # the sum overflows
    assert median_bits([2.5], F64) == fb(2.5) and median_bits([], F64) is None
    assert median_bits([3.25] * 6, F64) == fb(3.25) and median_bits([-7] * 5, I64) == (-7) & M64


def test_row_selection():
    """NULLs, time ranges, predicates on another column, column tombstones and buckets."""
    ts = np.arange(10, dtype=np.int64) * 10
    v = np.array([5, 1, 9, 3, 7, 2, 8, 6, 4, 0], dtype=np.int64)
    ok = np.array([1, 1, 0, 1, 1, 1, 1, 1, 1, 1], dtype=bool)
    w = np.arange(10, dtype=np.float64)
    truth = {0: [(ts, {1: (v, ok), 2: (w, np.ones(10, dtype=bool))})]}
    q = QueryOption([PushedAggregate(1, I64, ["median"])], width=50, first_bucket_start=0, n_buckets=2,
                    time_ranges=[(10, 80)], predicates=[(2, F64, "!=", 4.0)])
    cells = selected_values(truth, q, 1, I64)
    assert cells == {0: [1, 3], 1: [2, 8, 6, 4]}  # (row 2 NULL, row 4 filtered; ranges are closed)
    vals, valid = exact_median_cells(truth, q, 1, I64, 2)
    assert list(valid) == [True, True] and list(vals) == [2, 5]
    tombs = cabi.tombstones([(0, 1, 0, 25)])
    assert selected_values(truth, q, 1, I64, tombstones=tombs) == {0: [3], 1: [2, 8, 6, 4]}
