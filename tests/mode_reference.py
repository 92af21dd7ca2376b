"""Exact per-cell mode(x) and COUNT(DISTINCT x) (TSKV_QUERY_N_MODES / _N_DISTINCTS) for arenas described by a `truth`
dict (tests/helpers.py random_arena's), with median_reference.selected_values' row selection.

Two values are equal iff their bit patterns are (f64: -0.0 and +0.0 differ, NaNs are equal only with equal bits), as
ModeAccumulator's HashMap<ScalarValue, u32> counts them. The mode is the value that occurs most often; of tied values it
is the smallest in the type's order (f64: IEEE totalOrder), the engine's documented tie rule (the reference picks any
tied value). The distinct count is the number of distinct bit patterns, 0 in a cell without a value."""
import json
import os
from collections import Counter

import numpy as np

from cnosdb_b200 import cabi
from tests.median_reference import bits_of, f64_key, selected_values


def order_key(bits, pt):
    """The type's order of a u64 bit pattern (f64: totalOrder)."""
    if pt == cabi.TSKV_PT_F64:
        return f64_key(bits)
    if pt == cabi.TSKV_PT_I64:
        return bits - (1 << 64) if bits >> 63 else bits
    return bits


def mode_bits(values, pt):
    """(the mode as a u64 bit pattern or None for no value, the number of distinct values) of typed values."""
    counts = Counter(bits_of(v, pt) for v in values)
    if not counts:
        return None, 0
    best = max(counts.values())
    return min((b for b, n in counts.items() if n == best), key=lambda b: order_key(b, pt)), len(counts)


def exact_mode_cells(truth, query, col, pt, n_cells, **kw):
    """(mode bit patterns u64 [n_cells], mode validity bool [n_cells], distinct counts u64 [n_cells]) of (col, pt)."""
    v = np.zeros(n_cells, dtype=np.uint64)
    ok = np.zeros(n_cells, dtype=bool)
    nd = np.zeros(n_cells, dtype=np.uint64)
    for cell, vals in selected_values(truth, query, col, pt, **kw).items():
        m, d = mode_bits(vals, pt)
        nd[cell] = d
        if m is not None:
            v[cell], ok[cell] = m, True
    return v, ok, nd


def check_mode(res, j, exact, what=""):
    """Output j of a ScanResult, a mode, against exact_mode_cells: validity equal, values bit for bit."""
    v_e, ok_e, _ = exact
    v, ok = res.values[j], res.validity[j]
    np.testing.assert_array_equal(ok, ok_e, err_msg=what + " mode validity")
    bad = np.nonzero(ok_e & (v != v_e))[0]
    assert bad.size == 0, (what, [(int(i), hex(int(v[i])), hex(int(v_e[i]))) for i in bad[:5]])


def check_distinct(res, j, exact, what=""):
    """Output j of a ScanResult, a distinct count, against exact_mode_cells: always valid, counts equal."""
    assert res.validity[j].all(), what + " distinct validity"
    np.testing.assert_array_equal(res.values[j], exact[2], err_msg=what + " distinct")


GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "mode_slt.json")
PT_OF = {"BIGINT": cabi.TSKV_PT_I64, "BIGINT UNSIGNED": cabi.TSKV_PT_U64, "DOUBLE": cabi.TSKV_PT_F64}


class GoldenCase:
    """One answer of mode.slt / approx_distinct.slt over its table: rows (time ns, series tags, value or None), the
    predicate `value == pred` of a WHERE x IN (v) (or None), the tag whose values group the rows (or None), the kind
    ("mode" / "distinct") and the expected answer of each group in tag order."""

    def __init__(self, what, kind, pt, rows, expected, group_tag=None, pred=None):
        self.what, self.kind, self.pt, self.rows = what, kind, pt, rows
        self.expected, self.group_tag, self.pred = expected, group_tag, pred

    def groups(self):
        """{group key: [selected values]} in group-key order."""
        out = {}
        for _, tags, v in self.rows:
            key = tags[self.group_tag] if self.group_tag is not None else ""
            vals = out.setdefault(key, [])
            if v is not None and (self.pred is None or v == self.pred):
                vals.append(v)
        return dict(sorted(out.items()))


def _ns(s):
    return int(np.datetime64(s.replace(" ", "T"), "ns").astype(np.int64))


def _value(s, pt):
    if s.upper() == "NULL":
        return None
    return float(s) if pt == cabi.TSKV_PT_F64 else int(s)


def golden_cases():
    """The GoldenCases of tests/golden/mode_slt.json."""
    with open(GOLDEN) as f:
        g = json.load(f)
    cases = []
    tbl = g["func_tbl"]
    cols = tbl["columns"]
    raw = tbl["setup"]["rows"] + tbl["mode_insert"]["rows"]

    def func_tbl_rows(col):
        pt = PT_OF[tbl["types"][col]]
        return pt, [(_ns(r[0]), (r[cols.index("t0")], r[cols.index("t1")]), _value(r[cols.index(col)], pt)) for r in raw]
    for a in g["func_tbl_modes"]:
        pt, rows = func_tbl_rows(a["column"])
        cases.append(GoldenCase(a["src"], "mode", pt, rows, [a["expected"]]))
    a = g["func_tbl_mode_by_t0"]
    pt, rows = func_tbl_rows(a["column"])
    cases.append(GoldenCase(a["src"], "mode", pt, rows, a["expected"], group_tag=0))
    tb3 = g["func_tb3"]
    for a in g["func_tb3_modes"]:
        pt = PT_OF[tb3["types"][a["column"]]]
        conv = float if pt == cabi.TSKV_PT_F64 else int
        rows = [(_ns(r["time"]), (r["t0"],), conv(r[a["column"]])) for r in tb3["rows"]]
        cases.append(GoldenCase(a["src"], "mode", pt, rows, [conv(a["expected"])], pred=conv(a["in"])))
    nulls = g["tbl_with_nulls"]
    for a in g["distinct"]:
        pt = PT_OF[nulls["types"][a["column"]]]
        j = nulls["columns"].index(a["column"])
        rows = [(_ns(r[0]), (), _value(r[j], pt)) for r in nulls["rows"]]
        cases.append(GoldenCase(a["src"], "distinct", pt, rows, [a["expected"]]))
    return cases


def golden_refused():
    """The operand types mode.slt answers that the scan refuses: [(column, type, src)]."""
    with open(GOLDEN) as f:
        return [(r["column"], r["type"], r["src"]) for r in json.load(f)["refused"]]
