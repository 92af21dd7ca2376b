"""Exact per-cell counter increases (TSKV_QUERY_N_INCREASES) for arenas described by a `truth` dict (tests/helpers.py
random_arena's: truth[series] = [(ts, {column: (values, valid)}), ...] per column group).

The row selection is covariance_reference.paired_rows' with one operand, as median_reference composes it: the operand is
paired with a row-number column that is valid wherever the operand is, so a row counts when its series is selected, its
timestamp lies in the query's time ranges and in a bucket, the AND-ed predicates hold, no row-drop tombstone covers it,
and the operand is valid and not masked by a column tombstone (with `files`, the merged rows of overlapping chunks).

A cell's selected values are walked in time order (IncreaseAccumulator::update_inner): each value v after the previous
one `last` adds v - last when v > last, v when v < last (a counter reset) and nothing when they are equal, in the type's
order (i64 signed, u64 unsigned, f64 IEEE totalOrder on the bit pattern); the sum starts at 0. Integers subtract and add
wrapping at 64 bits; f64 adds sequentially in time order (the scan adds in atomic order: check_increase compares f64
sums within the SUM rules)."""
import numpy as np

from cnosdb_b200 import cabi
from tests.covariance_reference import paired_rows
from tests.median_reference import bits_of, f64_key

ROW = -1  # the row-number column paired with the operand (no column id of an arena)
MASK = 0xFFFFFFFFFFFFFFFF


def order_key(bits, pt):
    """The order key of a u64 bit pattern of type pt."""
    if pt == cabi.TSKV_PT_F64:
        return f64_key(bits)
    if pt == cabi.TSKV_PT_I64:
        return bits - (1 << 64) if bits >> 63 else bits
    return bits


def increase_bits(values, pt):
    """(u64 bit pattern of the increase of typed values in time order, sum of |contributions| for f64), or (None, 0.0)
    for no value."""
    if len(values) == 0:
        return None, 0.0
    b = [bits_of(v, pt) for v in values]
    if pt == cabi.TSKV_PT_F64:
        acc, mag = 0.0, 0.0
        for last, v in zip(b, b[1:]):
            kl, kv = f64_key(last), f64_key(v)
            x, y = (float(np.uint64(u).view(np.float64)) for u in (v, last))
            d = 0.0 if kv == kl else (x - y if kv > kl else x)
            acc += d
            mag += abs(d)
        return bits_of(acc, pt), mag
    acc = 0
    for last, v in zip(b, b[1:]):
        kl, kv = order_key(last, pt), order_key(v, pt)
        if kv > kl:
            acc = (acc + v - last) & MASK
        elif kv < kl:
            acc = (acc + v) & MASK
    return acc, 0.0


def selected_rows(truth, query, col, pt, **kw):
    """{cell: [(time, typed value)]} of operand (col, pt) under `query`, in time order, with paired_rows' selection
    (tombstones, group_ids, edges, labels, files as there)."""
    ids, flat, flat_t = {}, [], []
    for sid, cgs in truth.items():
        out = []
        for ts, cols in cgs:
            if col in cols:
                v, ok = cols[col]
                rows = np.arange(len(flat), len(flat) + len(v), dtype=np.int64)
                flat.extend(v)
                flat_t.extend(int(t) for t in ts)
                cols = dict(cols)
                cols[ROW] = (rows, np.asarray(ok, dtype=bool))
            out.append((ts, cols))
        ids[sid] = out
    cells = paired_rows(ids, query, (col, pt, ROW, cabi.TSKV_PT_I64), **kw)
    return {cell: sorted(((flat_t[int(r)], flat[int(r)]) for r in rows), key=lambda p: p[0])
            for cell, (_, rows) in cells.items()}


def exact_increase_cells(truth, query, col, pt, n_cells, **kw):
    """(bit patterns u64 [n_cells], validity bool [n_cells], f64 magnitudes [n_cells]) of the increase of (col, pt)."""
    v = np.zeros(n_cells, dtype=np.uint64)
    ok = np.zeros(n_cells, dtype=bool)
    mag = np.zeros(n_cells, dtype=np.float64)
    for cell, rows in selected_rows(truth, query, col, pt, **kw).items():
        x, m = increase_bits([r[1] for r in rows], pt)
        if x is not None:
            v[cell], ok[cell], mag[cell] = x, True, m
    return v, ok, mag


def increase_cells_np(cells, times, bits, pt, n_cells):
    """The increase of every cell over selected rows given as arrays (cell index, time, u64 bit pattern per row; a cell
    holds rows of one series, at distinct times), vectorized for page sets too large for exact_increase_cells -> the
    same (bit patterns u64 [n_cells], validity bool [n_cells], f64 magnitudes [n_cells]). Integers sum in uint64
    (wrapping); f64 contributions sum in row order, which check_increase's tolerance covers."""
    cells = np.asarray(cells, dtype=np.int64)
    bits = np.asarray(bits, dtype=np.uint64)
    order = np.lexsort((np.asarray(times, dtype=np.int64), cells))
    c, b = cells[order], bits[order]
    ok = np.zeros(n_cells, dtype=bool)
    ok[c] = True
    v = np.zeros(n_cells, dtype=np.uint64)
    mag = np.zeros(n_cells, dtype=np.float64)
    pair = c[1:] == c[:-1]
    last, cur, pc = b[:-1][pair], b[1:][pair], c[1:][pair]
    if pt == cabi.TSKV_PT_F64:
        neg = (1 << 63)
        key = lambda u: np.where(u >> np.uint64(63), ~u, u | np.uint64(neg))  # noqa: E731  (totalOrder, unsigned)
        kl, kv = key(last), key(cur)
        x, y = cur.view(np.float64), last.view(np.float64)
        with np.errstate(invalid="ignore", over="ignore"):
            d = np.where(kv == kl, 0.0, np.where(kv > kl, x - y, x))
            acc = np.zeros(n_cells, dtype=np.float64)
            np.add.at(acc, pc, d)
            np.add.at(mag, pc, np.abs(d))
        return acc.view(np.uint64), ok, mag
    if pt == cabi.TSKV_PT_I64:
        kl, kv = last.view(np.int64), cur.view(np.int64)
    else:
        kl, kv = last, cur
    d = np.where(kv == kl, np.uint64(0), np.where(kv > kl, cur - last, cur))
    np.add.at(v, pc, d)
    return v, ok, mag


def check_increase(res, j, exact, pt, what=""):
    """Output j of a ScanResult, an increase, against exact_increase_cells: validity equal; integers bit for bit; f64
    NaN where the reference has NaN, +-inf equal, finite values within 1e-12 of the contributions' magnitude (the sum's
    order is atomic order, as for SUM)."""
    v_e, ok_e, mag = exact
    v, ok = res.values[j], res.validity[j]
    np.testing.assert_array_equal(ok, ok_e, err_msg=what + " increase validity")
    if pt != cabi.TSKV_PT_F64:
        bad = np.nonzero(ok_e & (v != v_e))[0]
        assert bad.size == 0, (what, [(int(i), hex(int(v[i])), hex(int(v_e[i]))) for i in bad[:5]])
        return
    x, y = v.view(np.float64)[ok_e], v_e.view(np.float64)[ok_e]
    np.testing.assert_array_equal(np.isnan(x), np.isnan(y), err_msg=what + " increase NaN")
    fin = np.isfinite(y)
    np.testing.assert_array_equal(x[~fin & ~np.isnan(y)], y[~fin & ~np.isnan(y)], err_msg=what + " increase inf")
    err = np.abs(x[fin] - y[fin])
    tol = 1e-12 * mag[ok_e][fin] + 1e-300
    assert (err <= tol).all(), (what, x[fin][err > tol][:5], y[fin][err > tol][:5])


# ---- the reference's increase goldens (tests/golden/increase_slt.json, written by tests/golden/make_increase_golden.py) ----
def load_golden():
    import json
    import os
    with open(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "increase_slt.json")) as f:
        return json.load(f)
