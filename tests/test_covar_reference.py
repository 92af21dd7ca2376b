"""The host formulas of the column pairs (engine.pair_stat) on exact co-moments (tests/covariance_reference.py), no GPU:
DataFusion's covar / covar_samp / covar_pop / corr, the corr = 0.0 rule of a constant column, the n = 0 / 1 rules, and
data whose exact covariance is 0 (DataFusion's online update leaves a rounding residue there; the two-pass scan gives
0.0). The goldens are the reference's corr / covar / covar_pop / covar_samp checks (tests/golden/covar_slt.json)."""
import math

import numpy as np
import pytest

from cnosdb_b200.engine import pair_stat
from tests.covariance_reference import exact_comoments, load_golden, tb2_column


def stats(xs, ys, name):
    n, c, m2x, m2y = exact_comoments(xs, ys)
    v, ok = pair_stat(name, [n], [0.0 if c is None else c], [0.0 if m2x is None else m2x], [0.0 if m2y is None else m2y], [n > 0])
    return float(v[0]) if ok[0] else None


def test_textbook_values():
    xs, ys = [1.0, 2.0, 3.0, 4.0], [2.0, 4.0, 6.0, 9.0]
    mx, my = np.mean(xs), np.mean(ys)
    c = sum((a - mx) * (b - my) for a, b in zip(xs, ys))
    assert stats(xs, ys, "covar") == pytest.approx(c / 3, rel=1e-15)
    assert stats(xs, ys, "covar_samp") == stats(xs, ys, "covar")
    assert stats(xs, ys, "covar_pop") == pytest.approx(c / 4, rel=1e-15)
    assert stats(xs, ys, "corr") == pytest.approx(np.corrcoef(xs, ys)[0, 1], rel=1e-14)
    assert stats(xs, [-y for y in ys], "corr") == pytest.approx(-np.corrcoef(xs, ys)[0, 1], rel=1e-14)
    assert stats(xs, xs, "corr") == pytest.approx(1.0, rel=1e-15)


def test_constant_column_gives_zero():
    assert stats([1.0, 1.0, 1.0], [2.0, 5.0, 7.0], "corr") == 0.0
    assert stats([3.5] * 5, [3.5] * 5, "corr") == 0.0
    assert stats([1.0], [2.0], "corr") == 0.0  # corr(1, 2) = 0.0 on one row
    assert stats([1e9 + 0.25] * 7, [2.0, 1.0, 0.0, 5.0, 1.0, 1.0, 3.0], "covar_pop") == 0.0


def test_empty_and_single_row():
    for name in ("covar", "covar_samp", "covar_pop", "corr"):
        assert stats([], [], name) is None
    assert stats([4.0], [7.0], "covar") is None and stats([4.0], [7.0], "covar_samp") is None
    assert stats([4.0], [7.0], "covar_pop") == 0.0


def test_exactly_uncorrelated_is_zero():
    # x symmetric around its mean against y even in the same offsets: the exact co-moment is 0
    xs = [1.0, 2.0, 3.0, 4.0, 5.0, 6.0, 7.0]
    ys = [0.1, 0.7, 0.3, 0.9, 0.3, 0.7, 0.1]
    assert exact_comoments(xs, ys)[1] == 0.0
    assert stats(xs, ys, "covar") == 0.0 and stats(xs, ys, "corr") == 0.0


def test_integer_extremes_and_specials():
    xs = [float(2**63 - 1), float(-2**63), 0.0, 12345.0]
    ys = [float(2**64 - 1), 0.0, float(2**63), 1.0]
    n, c, m2x, m2y = exact_comoments(xs, ys)
    assert n == 4 and math.isfinite(c) and m2x > 0 and m2y > 0
    n, c, m2x, m2y = exact_comoments([1.0, math.nan], [1.0, 2.0])
    assert math.isnan(c) and math.isnan(m2x) and m2y == 0.5
    v, ok = pair_stat("corr", [2], [c], [m2x], [m2y], [True])
    assert ok[0] and math.isnan(v[0])


# ---- the reference's goldens (tests/golden/covar_slt.json) -------------------------------------------------------------
G = load_golden()


def golden_stat(func, xs, ys):
    n, c, m2x, m2y = exact_comoments(list(np.asarray(xs, dtype=np.float64)), list(np.asarray(ys, dtype=np.float64)))
    v, ok = pair_stat(func, [n], [0.0 if c is None else c], [0.0 if m2x is None else m2x], [0.0 if m2y is None else m2y], [n > 0])
    return float(v[0]) if ok[0] else None


def test_golden_extraction():
    assert len(G["checks"]) == 20 and len(G["constants"]) == 4 and len(G["nulls"]) == 4 and len(G["refused"]) == 8
    assert len(G["unorder"]["rows"]) == 10 and len(G["unorder"]["expected"]) == 12
    assert {c["func"] for c in G["checks"]} == {"corr", "covar", "covar_pop", "covar_samp"}
    for c in G["checks"] + G["constants"] + G["nulls"] + G["refused"] + G["unorder"]["expected"]:
        path, line = c["src"].rsplit(":", 1)
        assert path.endswith(".slt") and int(line) > 0, c


@pytest.mark.parametrize("i", range(20))
def test_golden_checks(i):
    """abs(F(a, b) - v) < tol of corr.slt / covar*.slt, from the exact co-moments of func_tb2's operands."""
    c = G["checks"][i]
    got = golden_stat(c["func"], tb2_column(G, c["x"]), tb2_column(G, c["y"]))
    assert got is not None and abs(got - c["value"]) < c["tolerance"], (c, got)


def test_golden_constants_and_nulls():
    n = len(G["tables"]["func_tb2"]["rows"])
    for c in G["constants"]:  # F(1, 2) over every row: constant operands
        assert golden_stat(c["func"], [1.0] * n, [2.0] * n) == float(c["expected"]), c
    for c in G["nulls"]:  # F(f1, f3): the STRING f3 converts to no f64 value, so no row pairs -> NULL
        assert golden_stat(c["func"], [], []) is None, c


def test_golden_unorder_is_exactly_zero():
    """unorderdata_func.slt: DataFusion's online update leaves a rounding residue (6.28e-17 / 4.93e-17 / 4.44e-17) where the
    exact covariance is 0; the two-pass formulas give 0.0, within an absolute tolerance of the golden values."""
    rows = G["unorder"]["rows"]
    xs, ys = [float(r[1]) for r in rows], [float(r[2]) for r in rows]
    assert exact_comoments(xs, ys)[1] == 0.0
    for e in G["unorder"]["expected"]:
        got = golden_stat(e["func"], xs, ys)
        assert got == 0.0 and abs(got - e["value"]) < 1e-16, e
