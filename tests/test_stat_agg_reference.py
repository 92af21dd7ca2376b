"""The host half of var* / stddev* (engine.stat_from_m2) and the exact M2 of tests/variance_reference.py against the
reference's statistical_agg expectations (tests/golden/stat_agg_slt.json) and hand-worked cases. CPU only."""
import json
import math
import os

import numpy as np
import pytest

from cnosdb_b200 import cabi
from cnosdb_b200.engine import STAT_AGGS, PushedAggregate, stat_from_m2
from tests.variance_reference import as_f64, exact_m2

GOLDEN = json.load(open(os.path.join(os.path.dirname(__file__), "golden", "stat_agg_slt.json")))
PHYS = {"BIGINT": cabi.TSKV_PT_I64, "BIGINT UNSIGNED": cabi.TSKV_PT_U64, "DOUBLE": cabi.TSKV_PT_F64}


def column_f64(table, column):
    """The golden table's column as f64, through the u64 bit patterns the scan sees."""
    t = GOLDEN["tables"][table]
    pt = PHYS[t["types"][column]]
    j = t["columns"].index(column)
    raw = [r[j] for r in t["rows"]]
    if pt == cabi.TSKV_PT_F64:
        bits = np.array([float(x) for x in raw], dtype=np.float64).view(np.uint64)
    else:
        bits = np.array([int(x) & (2**64 - 1) for x in raw], dtype=np.uint64)
    return as_f64(pt, bits)


@pytest.mark.parametrize("check", GOLDEN["checks"], ids=lambda c: "%s-%s-%s" % (c["func"], c["table"], c["column"]))
def test_golden_within_threshold(check):
    x = column_f64(check["table"], check["column"])
    m2 = exact_m2(x)
    v, ok = stat_from_m2(check["func"], np.array([x.size]), np.array([m2]), np.array([True]))
    assert ok[0]
    assert abs(v[0] - check["value"]) < check["tolerance"], (check["src"], v[0])


def test_golden_covers_every_function_and_type():
    assert {c["func"] for c in GOLDEN["checks"]} == {"stddev_samp", "stddev_pop", "var", "var_pop", "var_samp"}
    assert {GOLDEN["tables"][c["table"]]["types"][c["column"]] for c in GOLDEN["checks"]} == set(PHYS)
    assert len(GOLDEN["checks"]) == 24


@pytest.mark.parametrize("case", GOLDEN["constants"], ids=lambda c: c["func"])
def test_golden_constant_argument(case):
    n = len(GOLDEN["tables"][case["table"]]["rows"])
    v, ok = stat_from_m2(case["func"], np.array([n]), np.array([exact_m2([1.0] * n)]), np.array([True]))
    assert ok[0] and v[0] == float(case["expected"])


def test_golden_refused_types_are_boolean_and_string():
    # the scan refuses M2 on BOOL columns (as SUM); string columns are not aggregated by it at all
    for r in GOLDEN["refused"]:
        assert GOLDEN["tables"][r["table"]]["types"].get(r["column"], "STRING") in ("BOOLEAN", "STRING"), r
    assert {r["type"] for r in GOLDEN["refused"]} == {"Boolean", "Utf8"}


def test_derived_names_request_count_and_m2():
    for name in STAT_AGGS:
        assert PushedAggregate(1, cabi.TSKV_PT_F64, [name]).agg_mask == cabi.TSKV_AGG_COUNT | cabi.TSKV_AGG_M2
    assert PushedAggregate(1, cabi.TSKV_PT_F64, ["mean", "stddev"]).agg_list() == [1, 16, 128]
    assert cabi.AGG_NAMES[cabi.TSKV_AGG_M2] == "m2" and cabi.TSKV_AGG_ALL == 0x7F


def test_exact_m2_small_cases():
    assert exact_m2([]) is None
    assert exact_m2([5.0]) == 0.0
    assert exact_m2([3.25] * 7) == 0.0
    assert exact_m2([1.0, 2.0, 3.0, 4.0]) == 5.0
    assert math.isnan(exact_m2([1.0, math.nan]))
    assert math.isnan(exact_m2([1.0, math.inf]))
    assert math.isnan(exact_m2([-math.inf, math.inf]))
    # ill-conditioned: 1e9 plus small offsets, where the naive sum of squares loses every digit
    xs = [1e9 + k * 1e-3 for k in range(5)]
    assert exact_m2(xs) == pytest.approx(sum((x - sum(xs) / 5) ** 2 for x in xs), rel=1e-6)


def test_exact_m2_integer_extremes_convert_to_f64_first():
    u = np.array([2**64 - 1, 2**63 + 1, 2**63], dtype=np.uint64)
    x = as_f64(cabi.TSKV_PT_U64, u)
    assert x.tolist() == [2.0**64, 2.0**63, 2.0**63]  # the cast rounds before any arithmetic
    mean = (2.0**64 + 2 * 2.0**63) / 3
    assert exact_m2(x) == pytest.approx((2.0**64 - mean) ** 2 + 2 * (2.0**63 - mean) ** 2, rel=1e-15)
    i = np.array([-2**63, 2**63 - 1], dtype=np.int64).view(np.uint64)
    x = as_f64(cabi.TSKV_PT_I64, i)
    assert x.tolist() == [-2.0**63, 2.0**63]
    assert exact_m2(x) == 2 * 2.0**126


def test_final_formulas():
    n = np.array([0, 1, 2, 4], dtype=np.uint64)
    m2 = np.array([0.0, 0.0, 2.0, 5.0])
    ok = n > 0
    v, good = stat_from_m2("var_pop", n, m2, ok)
    assert good.tolist() == [False, True, True, True] and v[1:].tolist() == [0.0, 1.0, 1.25]
    v, good = stat_from_m2("var_samp", n, m2, ok)  # one value: NULL (DESIGN.md section 7: not pinned by the reference)
    assert good.tolist() == [False, False, True, True] and v[2:].tolist() == [2.0, 5.0 / 3]
    v, good = stat_from_m2("stddev", n, m2, ok)
    assert good.tolist() == [False, False, True, True] and v[3] == math.sqrt(5.0 / 3)
    v, good = stat_from_m2("stddev_pop", n, np.array([0.0, 0.0, math.nan, 5.0]), ok)
    assert math.isnan(v[2]) and v[3] == math.sqrt(1.25)
