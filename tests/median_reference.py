"""Exact per-cell medians (TSKV_QUERY_N_MEDIANS) for arenas described by a `truth` dict (tests/helpers.py random_arena's:
truth[series] = [(ts, {column: (values, valid)}), ...] per column group).

The row selection is covariance_reference.paired_rows' with one operand: the operand is paired with a row-number column
that is valid wherever the operand is, so a row counts when its series is selected, its timestamp lies in the query's
time ranges and in a bucket of the grid (or of the edges), the AND-ed predicates hold, no row-drop tombstone covers it,
and the operand is valid and not masked by a column tombstone. The selected values of a cell are ordered by their
type's order (f64: IEEE totalOrder on the bit pattern, so NaN is a value and -0.0 < +0.0). For odd n the median is the
value at rank n // 2; for even n it is lo.add_wrapping(hi).div_wrapping(2) of the values at ranks n // 2 - 1 and n // 2 in
the operand's type: i64 wrapping add then division truncating toward zero, u64 wrapping add then // 2, f64 (lo + hi) /
2.0 with x86-64 SSE NaN results (a NaN operand's bits quieted, lo first; -inf + inf is 0xfff8000000000000), spelled out
here so that the result does not depend on the host's floating-point unit."""
import math

import numpy as np

from cnosdb_b200 import cabi
from tests.covariance_reference import paired_rows

ROW = -1  # the row-number column paired with the operand (no column id of an arena)
QUIET = 0x0008000000000000
DEFAULT_NAN = 0xFFF8000000000000


def f64_key(bits):
    """Signed order key of an f64 bit pattern (IEEE totalOrder), as the scan's MIN / MAX key."""
    bits = int(bits)
    k = bits ^ (0x7FFFFFFFFFFFFFFF if bits >> 63 else 0)
    return k - (1 << 64) if k >> 63 else k


def bits_of(v, pt):
    """The u64 bit pattern of one value of type pt."""
    if pt == cabi.TSKV_PT_F64:
        return int(np.float64(v).view(np.uint64))
    return int(v) & 0xFFFFFFFFFFFFFFFF


def median_bits(values, pt):
    """The median of typed values (bit patterns) as a u64 bit pattern, or None for no value."""
    n = len(values)
    if n == 0:
        return None
    b = [bits_of(v, pt) for v in values]
    if pt == cabi.TSKV_PT_F64:
        b.sort(key=f64_key)
    elif pt == cabi.TSKV_PT_I64:
        b.sort(key=lambda x: x - (1 << 64) if x >> 63 else x)
    else:
        b.sort()
    if n % 2:
        return b[n // 2]
    lo, hi = b[n // 2 - 1], b[n // 2]
    if pt == cabi.TSKV_PT_U64:
        return ((lo + hi) & 0xFFFFFFFFFFFFFFFF) // 2
    if pt == cabi.TSKV_PT_I64:
        s = (lo + hi) & 0xFFFFFFFFFFFFFFFF
        s = s - (1 << 64) if s >> 63 else s
        q = abs(s) // 2  # truncation toward zero
        return (q if s >= 0 else -q) & 0xFFFFFFFFFFFFFFFF
    x, y = (float(np.uint64(v).view(np.float64)) for v in (lo, hi))
    if math.isnan(x):
        return lo | QUIET
    if math.isnan(y):
        return hi | QUIET
    s = x + y
    if math.isnan(s):
        return DEFAULT_NAN
    return bits_of(s / 2.0, pt)


def selected_values(truth, query, col, pt, **kw):
    """{cell: [typed values]} of operand (col, pt) under `query`, with paired_rows' selection (tombstones, group_ids,
    edges, labels as there)."""
    ids, flat = {}, []
    for sid, cgs in truth.items():
        out = []
        for ts, cols in cgs:
            if col in cols:
                v, ok = cols[col]
                rows = np.arange(len(flat), len(flat) + len(v), dtype=np.int64)
                flat.extend(v)
                cols = dict(cols)
                cols[ROW] = (rows, np.asarray(ok, dtype=bool))
            out.append((ts, cols))
        ids[sid] = out
    cells = paired_rows(ids, query, (col, pt, ROW, cabi.TSKV_PT_I64), **kw)
    return {cell: [flat[int(r)] for r in rows] for cell, (_, rows) in cells.items()}


def exact_median_cells(truth, query, col, pt, n_cells, **kw):
    """(bit patterns u64 [n_cells], validity bool [n_cells]) of the median of (col, pt)."""
    v = np.zeros(n_cells, dtype=np.uint64)
    ok = np.zeros(n_cells, dtype=bool)
    for cell, vals in selected_values(truth, query, col, pt, **kw).items():
        m = median_bits(vals, pt)
        if m is not None:
            v[cell], ok[cell] = m, True
    return v, ok


def check_median(res, j, exact, what=""):
    """Output j of a ScanResult, a median, against exact_median_cells: validity equal, values bit for bit."""
    v_e, ok_e = exact
    v, ok = res.values[j], res.validity[j]
    np.testing.assert_array_equal(ok, ok_e, err_msg=what + " median validity")
    bad = np.nonzero(ok_e & (v != v_e))[0]
    assert bad.size == 0, (what, [(int(i), hex(int(v[i])), hex(int(v_e[i]))) for i in bad[:5]])
