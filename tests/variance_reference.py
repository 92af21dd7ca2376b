"""Exact M2 (TSKV_AGG_M2: the sum of squared deviations from the cell mean) for the exact references of tests/helpers.py.

The cells come from the reference that runs: exact_aggregate, or its edges / labels / GROUP BY tags variants, which swap
the bucket rule and keep everything else. While it runs, the two calls its per-column tail makes on the final cell list
and values (np.bincount(cells) and _okey(pt, values)) are recorded; M2 of every cell is then computed with
fractions.Fraction over the values converted to f64, which is what the scan converts them to. NaN or +-inf among a cell's
values gives NaN."""
import contextlib
import math
from fractions import Fraction

import numpy as np

from cnosdb_b200 import cabi
from tests import helpers


def exact_m2(values_f64):
    """M2 = sum (x - mean)^2 of f64 values, exactly, rounded once to f64 (NaN with a NaN or infinite value; 0.0 for one
    value; None for none)."""
    xs = [float(x) for x in values_f64]
    if not xs:
        return None
    if not all(math.isfinite(x) for x in xs):
        return math.nan
    # x = p / q with q a power of two: on the common denominator Q every value is an integer k, and
    # M2 = (n * sum k^2 - (sum k)^2) / (n * Q^2) exactly
    ratios = [x.as_integer_ratio() for x in xs]
    big_q = max(q for _, q in ratios)
    ks = [p * (big_q // q) for p, q in ratios]
    n, s1, s2 = len(ks), sum(ks), sum(k * k for k in ks)
    try:
        return float(Fraction(n * s2 - s1 * s1, n * big_q * big_q))
    except OverflowError:
        return math.inf


def as_f64(pt, v):
    """u64 bit patterns of physical type pt -> f64, as (double)x."""
    v = np.asarray(v, dtype=np.uint64)
    if pt == cabi.TSKV_PT_F64:
        return v.view(np.float64)
    if pt == cabi.TSKV_PT_I64:
        return v.view(np.int64).astype(np.float64)
    return v.astype(np.float64)


class _NpRecorder:
    """numpy for tests.helpers, recording the cell list of every np.bincount call."""

    def __init__(self, log):
        self._log = log

    def __getattr__(self, name):
        return getattr(np, name)

    def bincount(self, x, *a, **kw):
        self._log.append(np.array(x, dtype=np.int64))
        return np.bincount(x, *a, **kw)


@contextlib.contextmanager
def _recording(cells, values):
    saved_np, saved_okey = helpers.np, helpers._okey

    def okey(pt, v):
        values.append((pt, np.array(v).view(np.uint64)))
        return saved_okey(pt, v)
    helpers.np, helpers._okey = _NpRecorder(cells), okey
    try:
        yield
    finally:
        helpers.np, helpers._okey = saved_np, saved_okey


def with_m2(run, query, n_groups=None):
    """run() -> ExactResult of `query` (any exact reference built on exact_aggregate; GROUP BY tags: n_groups groups of
    query.n_buckets cells, one exact_aggregate call per group), with every "m2" output filled in: the exact M2 of the
    cell's values, valid iff the cell holds one."""
    cells, values = [], []
    with _recording(cells, values):
        res = run()
    n_cols = len(query.columns)
    assert len(cells) == len(values) and len(cells) % n_cols == 0
    nb = query.n_buckets
    n_cells = res.values.shape[1]
    per_col = {c.column_id: {} for c in query.columns}  # column -> {cell: [f64 values]}
    for i, (cl, (pt, v)) in enumerate(zip(cells, values)):
        call, col = divmod(i, n_cols)
        base = call * nb if n_groups is not None else 0
        x = as_f64(pt, v)
        d = per_col[query.columns[col].column_id]
        for k, xv in zip(cl.tolist(), x.tolist()):
            d.setdefault(base + k, []).append(xv)
    for j, (c, name) in enumerate(res.names):
        if name != "m2":
            continue
        out = np.zeros(n_cells, dtype=np.float64)
        ok = np.zeros(n_cells, dtype=bool)
        for k, xs in per_col[c].items():
            out[k], ok[k] = exact_m2(xs), True
        res.values[j], res.validity[j] = out.view(np.uint64), ok
    return res


def check_m2(got, exp, what, rtol=1e-9):
    """got's m2 outputs against the exact ones: validity equal, NaN where NaN, else within rtol relative (plus the
    rounding of a shift that is not exactly the mean, for cells whose M2 is 0)."""
    n_m2 = 0
    for j, (col, agg) in enumerate(got.names):
        if agg != "m2":
            continue
        n_m2 += 1
        gv, ev = got.validity[j], exp.validity[j]
        assert (gv == ev).all(), "%s col %s: m2 validity differs at %s" % (what, col, np.nonzero(gv != ev)[0][:5])
        g = got.values[j].view(np.float64)[ev]
        e = exp.values[j].view(np.float64)[ev]
        nan = np.isnan(e)
        assert (np.isnan(g) == nan).all(), "%s col %s: NaN cells differ" % (what, col)
        with np.errstate(invalid="ignore"):
            bad = np.nonzero(~nan & ~(np.abs(g - e) <= rtol * np.abs(e) + 1e-300))[0]
        assert bad.size == 0, "%s col %s m2 at cells %s: got %s exact %s" % (
            what, col, np.nonzero(ev)[0][bad[:3]], g[bad[:3]], e[bad[:3]])
        assert (got.values[j][~gv] == 0).all()
    assert n_m2
