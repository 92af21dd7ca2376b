"""Shared test helpers: random arenas, numpy brute-force aggregation, result comparison."""
import math

import numpy as np

from cnosdb_b200 import cabi, datagen
from cnosdb_b200.engine import PushedAggregate, QueryOption

ALL_AGGS = ("count", "sum", "min", "max", "mean", "first", "last")


def bucket_spec(t_lo, t_hi, width, origin=0):
    """first_bucket_start / n_buckets covering [t_lo, t_hi] for t >= origin % width - width (floor regime)."""
    o = origin % width if origin >= 0 else -((-origin) % width)
    start = t_lo - ((t_lo - o + width) % width)
    n = (t_hi - start) // width + 1
    return start, int(n)


def assert_results_equal(got, exp, rtol=1e-6, what=""):
    """got/exp: ScanResult. Integers, counts, min/max/first/last bit-exact; f64 sum/mean within rtol."""
    assert got.names == exp.names
    for j, (col, agg) in enumerate(got.names):
        gv, ev = got.validity[j], exp.validity[j]
        assert (gv == ev).all(), "%s validity differs for col %s %s at %s" % (what, col, agg, np.nonzero(gv != ev)[0][:5])
        g, e = got.values[j][ev], exp.values[j][ev]
        pt = got.phys[col]
        if agg == "mean" or (agg == "sum" and pt == cabi.TSKV_PT_F64):
            gf, ef = g.view(np.float64), e.view(np.float64)
            ok = np.abs(gf - ef) <= rtol * np.maximum(np.abs(ef), 1e-300)
            assert ok.all(), "%s col %s %s: max rel err %g" % (what, col, agg, np.max(np.abs(gf - ef) / np.maximum(np.abs(ef), 1e-300)))
        else:
            bad = np.nonzero(g != e)[0]
            assert bad.size == 0, "%s col %s %s differs at %s: got %s exp %s" % (what, col, agg, bad[:5], g[bad[:5]], e[bad[:5]])
        # invalid cells hold 0
        assert (got.values[j][~ev] == 0).all()


def random_arena(rng, n_series=40, n_points=300, fields=((1, cabi.TSKV_PT_I64), (2, cabi.TSKV_PT_F64)),
                 null_frac=0.0, t0=1_000_000, step=1000, jitter=0, ids=None, raw_frac=0.0, multi_cg=False):
    """Hand-built arena via the product writer; returns (arena, descs, truth) where truth[series] is a
    list of column groups (ts, {col: (values, valid)})."""
    b = datagen.ArenaBuilder()
    truth = {}
    ids = list(range(n_series)) if ids is None else list(ids)
    for sid in ids:
        n_cg = 2 if (multi_cg and rng.random() < 0.3) else 1
        t_start = t0
        for _ in range(n_cg):
            n = int(n_points if not multi_cg else rng.integers(1, n_points + 1))
            ts = t_start + np.arange(n, dtype=np.int64) * step
            if jitter:
                ts = ts + rng.integers(-jitter, jitter + 1, n)
            t_start = int(ts[-1]) + step
            fl, cols = [], {}
            for col, pt in fields:
                valid = rng.random(n) >= null_frac if null_frac else None
                if pt == cabi.TSKV_PT_F64:
                    vals = np.cumsum(rng.integers(-3, 4, n)).astype(np.float64) + (rng.random(n) if rng.random() < 0.5 else 0)
                elif pt == cabi.TSKV_PT_U64:
                    vals = np.cumsum(rng.integers(0, 5, n)).astype(np.uint64) + np.uint64(2**63 - 100)
                else:
                    vals = np.cumsum(rng.integers(-50, 51, n)).astype(np.int64)
                enc = None
                if raw_frac and rng.random() < raw_frac:
                    enc = datagen.encode_raw
                fl.append((col, pt, vals, valid, enc))
                cols[col] = (vals, np.ones(n, dtype=bool) if valid is None else valid)
            b.add_column_group(sid, ts, fl)
            truth.setdefault(sid, []).append((ts, cols))
    arena, descs = b.finish()
    return arena, descs, truth


def make_query(fields, aggs=ALL_AGGS, **kw):
    cols = [PushedAggregate(c, pt, aggs) for c, pt in fields]
    return QueryOption(cols, **kw)


# ---- exact reference ---------------------------------------------------------------------------------------------------
# Aggregates computed from the generated arrays themselves (no page is decoded), so they share nothing with the oracle or
# the kernels. Integer sums are exact Python ints; f64 sums come with an error bound that holds for any summation order.
# FIRST / LAST are not restated here: compare those with the oracle.

I64_MIN, I64_MAX = -2**63, 2**63 - 1
_U = 2.0 ** -53  # unit roundoff of f64


class ReferenceError(RuntimeError):
    def __init__(self, status):
        super().__init__("reference status %d (%s)" % (status, cabi.STATUS_NAMES.get(status, "?")))
        self.status = status


def wrap64(x):
    """Python int -> the int64 it wraps to."""
    x &= (1 << 64) - 1
    return x - (1 << 64) if x >> 63 else x


def sliding_window(t, window, slide, start_time, i=0):
    """`sliding_window` of time_window.rs:184-198: Rust `%` truncates like C (np.fmod), `+` / `-` / `*` wrap (int64).
    t: int or int64 array -> (start, end), of the same shape."""
    scalar = np.ndim(t) == 0
    t = np.atleast_1d(np.asarray(t, dtype=np.int64))
    w, s = np.full_like(t, window), np.full_like(t, slide)
    with np.errstate(over="ignore"):
        st = np.fmod(np.full_like(t, start_time), w)
        last_start = t - np.fmod(t - st + s, s)
        ws = last_start - np.full_like(t, i) * s
        we = ws + w
    return (int(ws[0]), int(we[0])) if scalar else (ws, we)


def floor_sliding_window(t, window, slide, start_time):
    """time_window.rs:151-182: the last window that starts at or before t."""
    s, e = sliding_window(t, window, slide, start_time)
    if not (s <= t < e):
        while t < s:
            s, e = wrap64(s - slide), wrap64(e - slide)
    return s, e


def ceil_sliding_window(t, window, slide, start_time):
    """time_window.rs:97-147: the first window that holds t, else the first after it."""
    s = e = None
    for i in range((window + slide - 1) // slide - 1, -1, -1):
        s, e = sliding_window(t, window, slide, start_time, i)
        if s <= t < e:
            return s, e
    if s is not None:
        while t >= e:
            s, e = wrap64(s + slide), wrap64(e + slide)
    return s, e


def bucket_index(t, query):
    """Bucket of every timestamp (int64 array) and whether it has one: the window start of `sliding_window(t, w, w,
    origin)` must lie on the grid first_bucket_start + k * w, 0 <= k < n_buckets. Unbucketed: bucket 0."""
    t = np.asarray(t, dtype=np.int64)
    if query.width <= 0:
        return np.zeros(t.size, dtype=np.int64), np.ones(t.size, dtype=bool)
    ws, _ = sliding_window(t, query.width, query.width, query.origin)
    w = np.int64(query.width)
    with np.errstate(over="ignore"):
        diff = ws - np.int64(query.first_bucket_start)
    idx = np.where(diff >= 0, diff // w, -1)
    ok = (diff >= 0) & (np.fmod(diff, w) == 0) & (idx < query.n_buckets)
    return idx, ok


def _typed(pt, v):
    return np.asarray(v, dtype=np.float64 if pt == cabi.TSKV_PT_F64 else np.uint64 if pt == cabi.TSKV_PT_U64 else np.int64)


def _cmp(pt, op, v, c):
    """`column <op> constant` is TRUE (f64: NaN compares unordered)."""
    v = _typed(pt, v)
    c = np.float64(c) if pt == cabi.TSKV_PT_F64 else np.uint64(int(c) & 0xFFFFFFFFFFFFFFFF) if pt == cabi.TSKV_PT_U64 else np.int64(c)
    return [v == c, (v < c) | (v > c), v < c, v <= c, v > c, v >= c][op]


def _okey(pt, v):
    """Ordered int64 key: signed compare of keys == typed compare (f64: totalOrder, so -0.0 < +0.0)."""
    b = _typed(pt, v).view(np.uint64)
    if pt == cabi.TSKV_PT_U64:
        return (b ^ np.uint64(1 << 63)).view(np.int64)
    if pt == cabi.TSKV_PT_F64:
        return (b ^ ((b.view(np.int64) >> 63).view(np.uint64) & np.uint64(I64_MAX))).view(np.int64)
    return b.view(np.int64)


def _okey_inv(pt, k):
    k = np.asarray(k, dtype=np.int64)
    if pt == cabi.TSKV_PT_U64:
        return k.view(np.uint64) ^ np.uint64(1 << 63)
    if pt == cabi.TSKV_PT_F64:
        return k.view(np.uint64) ^ ((k >> 63).view(np.uint64) & np.uint64(I64_MAX))
    return k.view(np.uint64)


def gamma(k):
    """Higham's gamma_k = k u / (1 - k u): |computed - exact| <= gamma_{n-1} * sum|x| for any order of n-1 additions."""
    return k * _U / (1 - k * _U)


class ExactResult:
    """Expected dense result: values[j, cell] (u64 bits) and validity[j, cell] like ScanResult. For f64 SUM / MEAN
    `center[j]` holds the exactly rounded value (math.fsum) and `bound[j]` the largest error any summation order makes."""

    def __init__(self, query, n_groups):
        self.names = query.output_names()
        self.n_groups, self.n_buckets = n_groups, query.n_buckets
        n_cells = n_groups * query.n_buckets
        self.values = np.zeros((len(self.names), n_cells), dtype=np.uint64)
        self.validity = np.zeros((len(self.names), n_cells), dtype=bool)
        self.center, self.bound = {}, {}
        self.phys = {c.column_id: c.phys_type for c in query.columns}
        self.exact_sums = {}  # column id -> {cell: (S, n)} of integer columns


def exact_aggregate(truth, query):
    """COUNT / SUM / MIN / MAX / MEAN of `query` over `truth` ({series id: [(timestamps, {column id: (values,
    validity)}), ...]}, one entry per column group). Raises ReferenceError(TSKV_ERR_BUCKET_RANGE) when a selected row
    (time ranges, AND-ed predicates) has no bucket. A column group that holds none of the query columns is never read."""
    slots = [int(s) for s in query.series_ids] if query.series_ids is not None else sorted(truth)
    n_groups = len(slots) if query.group_by_series else 1
    nb = query.n_buckets
    n_cells = n_groups * nb
    qcols = [c.column_id for c in query.columns]
    cells = {c: [] for c in qcols}
    vals = {c: [] for c in qcols}
    for slot, sid in enumerate(slots):
        for ts, cols in truth.get(sid, []):
            if not any(c in cols for c in qcols):
                continue
            ts = np.asarray(ts, dtype=np.int64)
            sel = np.ones(ts.size, dtype=bool)
            for pc, ppt, op, c in query.predicates:  # NULL or an absent column: the comparison is not TRUE
                if pc not in cols:
                    sel[:] = False
                else:
                    pv, pvalid = cols[pc]
                    sel &= np.asarray(pvalid, dtype=bool) & _cmp(ppt, op, pv, c)
            if query.time_ranges:
                inr = np.zeros(ts.size, dtype=bool)
                for a, b in query.time_ranges:
                    inr |= (ts >= a) & (ts <= b)
                sel &= inr
            idx, ok = bucket_index(ts, query)
            if (sel & ~ok).any():
                raise ReferenceError(cabi.TSKV_ERR_BUCKET_RANGE)
            cell = (slot if query.group_by_series else 0) * nb + idx
            for c in qcols:
                if c in cols:
                    v, valid = cols[c]
                    m = sel & np.asarray(valid, dtype=bool)
                    cells[c].append(cell[m])
                    vals[c].append(np.asarray(v)[m])
    res = ExactResult(query, n_groups)
    j = 0
    for qc in query.columns:
        c, pt = qc.column_id, qc.phys_type
        cl = np.concatenate(cells[c]) if cells[c] else np.zeros(0, dtype=np.int64)
        v = _typed(pt, np.concatenate(vals[c]) if vals[c] else [])
        count = np.bincount(cl, minlength=n_cells).astype(np.uint64)
        have = count > 0
        out = {"count": (count, np.ones(n_cells, dtype=bool))}
        kmin = np.full(n_cells, I64_MAX, dtype=np.int64)
        kmax = np.full(n_cells, I64_MIN, dtype=np.int64)
        keys = _okey(pt, v)
        np.minimum.at(kmin, cl, keys)
        np.maximum.at(kmax, cl, keys)
        out["min"] = (np.where(have, _okey_inv(pt, kmin), 0).astype(np.uint64), have)
        out["max"] = (np.where(have, _okey_inv(pt, kmax), 0).astype(np.uint64), have)
        sums = np.zeros(n_cells, dtype=np.uint64)
        means = np.zeros(n_cells, dtype=np.uint64)
        live = np.nonzero(have)[0]
        if pt == cabi.TSKV_PT_F64:
            order = np.argsort(cl, kind="stable")
            parts = np.split(v[order], np.cumsum(count)[:-1].astype(np.int64))
            fs, ab = np.zeros(n_cells), np.zeros(n_cells)
            for k in live:
                fs[k] = math.fsum(parts[k])
                ab[k] = math.fsum(np.abs(parts[k]))
            n = count.astype(np.float64)
            # fsum is the exactly rounded sum: half an ulp more than gamma_{n-1} for the exact one
            sb = gamma(np.maximum(n - 1, 0)) * ab * (1 + 2 * _U) + _U * np.abs(fs)
            cen_mean = np.where(have, fs / np.maximum(n, 1), 0.0)
            sums = fs.view(np.uint64).copy()
            means = cen_mean.view(np.uint64).copy()
            res_f64 = {"sum": (fs, sb), "mean": (cen_mean, sb / np.maximum(n, 1) + 2 * _U * np.abs(cen_mean))}
        else:
            # exact S from the 32-bit halves: |sum of halves| < 2^63 for < 2^31 rows per cell
            b = v.view(np.uint64)
            lo = (b & np.uint64(0xFFFFFFFF)).astype(np.int64)
            hi = (v.view(np.int64) >> 32) if pt == cabi.TSKV_PT_I64 else (b >> np.uint64(32)).astype(np.int64)
            slo = np.zeros(n_cells, dtype=np.int64)
            shi = np.zeros(n_cells, dtype=np.int64)
            np.add.at(slo, cl, lo)
            np.add.at(shi, cl, hi)
            res.exact_sums[c] = {}
            for k in live:
                S = int(shi[k]) * 2**32 + int(slo[k])
                res.exact_sums[c][int(k)] = (S, int(count[k]))
                sums[k] = S % 2**64
                means[k] = np.float64(float(S) / float(int(count[k]))).view(np.uint64)
            res_f64 = {}
        out["sum"] = (sums, have)
        out["mean"] = (means, have)
        for a in qc.agg_list():
            name = cabi.AGG_NAMES[a]
            if name in out:
                res.values[j], res.validity[j] = out[name]
                if name in res_f64:
                    res.center[j], res.bound[j] = res_f64[name]
            j += 1
    return res


def assert_matches_exact(got, exp, what="", int_mean=True):
    """got: ScanResult; exp: ExactResult. COUNT / integer SUM / MIN / MAX bit-exact, integer MEAN bit-exact
    (= float(S) / float(n)) unless int_mean=False, f64 SUM / MEAN within the bound. FIRST / LAST are not checked."""
    assert got.names == exp.names
    for j, (col, agg) in enumerate(got.names):
        if agg in ("first", "last") or (agg == "mean" and not int_mean and exp.phys[col] != cabi.TSKV_PT_F64):
            continue
        gv, ev = got.validity[j], exp.validity[j]
        bad = np.nonzero(gv != ev)[0]
        assert bad.size == 0, "%s col %s %s: validity differs at cells %s" % (what, col, agg, bad[:5])
        if j in exp.center:
            g = got.values[j].view(np.float64)[ev]
            err = np.abs(g - exp.center[j][ev])
            bad = np.nonzero(~(err <= exp.bound[j][ev]))[0]
            assert bad.size == 0, "%s col %s %s: got %s, exact %s, bound %s" % (
                what, col, agg, g[bad[:3]], exp.center[j][ev][bad[:3]], exp.bound[j][ev][bad[:3]])
        else:
            g, e = got.values[j][ev], exp.values[j][ev]
            bad = np.nonzero(g != e)[0]
            assert bad.size == 0, "%s col %s %s differs at %s: got %s exp %s" % (
                what, col, agg, np.nonzero(ev)[0][bad[:5]], g[bad[:5]], e[bad[:5]])
        assert (got.values[j][~gv] == 0).all()


# ---- bucket-geometry sweep ---------------------------------------------------------------------------------------------
# Small arenas whose time geometry reaches the edges of the fused scan's bucket arithmetic. Each holds three blocks of 40
# series with fields i64 (simple8b walk), f64 (Gorilla) and u64:
#   A (ids 0-39)    identical RLE timestamps: whole warps agree and run the uniform bucket schedule;
#   B (ids 40-79)   RLE timestamps starting sid % 7 rows later, of varied lengths: the per-lane segment loop;
#   C (ids 80-119)  jittered timestamps (simple8b time pages for steps >= 2): locate_bucket per segment.
# Series 6, 19, ... hold nulls; series 45's i64 and f64 pages hold nothing but nulls.

GEOM_FIELDS = ((1, cabi.TSKV_PT_I64), (2, cabi.TSKV_PT_F64), (3, cabi.TSKV_PT_U64))
GEOM_BLOCK = 40
GEOM_SERIES = 3 * GEOM_BLOCK
GEOM_AGGS = ("count", "sum", "min", "max", "mean")
ALL_NULL_SERIES = 45


def geometry_timestamps(rng, sid, t0, step, n):
    """Timestamps of series `sid`: every row lies in [t0, t0 + (n - 1) * step] (Python ints, no wrap)."""
    span = (n - 1) * step
    blk = sid // GEOM_BLOCK
    if blk == 0:
        off = np.arange(n, dtype=np.uint64) * np.uint64(step)
    elif blk == 1:
        start = sid % 7 if n > 14 else 0
        m = n - start - (sid % 5) * (n // 9)  # >= 2 rows when n >= 2
        off = (np.arange(m, dtype=np.uint64) + np.uint64(start)) * np.uint64(step)
    else:
        # row k at k * step + [0, step): distinct, increasing times; the first and last row keep the geometry's extremes
        jit = rng.integers(0, max(step, 1), n, dtype=np.uint64)
        jit[0] = jit[-1] = 0
        off = np.arange(n, dtype=np.uint64) * np.uint64(step) + jit
    return (off + np.uint64(t0 % 2**64)).view(np.int64)  # t0 + off, exact: it stays in range


def geometry_arena(seed, t0, step, n):
    """-> (arena, descs, truth) of one sweep case (see above)."""
    rng = np.random.default_rng(seed)
    b = datagen.ArenaBuilder()
    truth = {}
    for sid in range(GEOM_SERIES):
        ts = geometry_timestamps(rng, sid, t0, step, n)
        m = ts.size
        fl, cols = [], {}
        for col, pt in GEOM_FIELDS:
            valid = rng.random(m) >= 0.3 if sid % 13 == 6 else np.ones(m, dtype=bool)
            if sid == ALL_NULL_SERIES and pt != cabi.TSKV_PT_U64:
                valid = np.zeros(m, dtype=bool)
            if pt == cabi.TSKV_PT_F64:
                vals = np.cumsum(rng.integers(-3, 4, m)).astype(np.float64) + rng.random(m)
            elif pt == cabi.TSKV_PT_U64:
                vals = np.cumsum(rng.integers(0, 5, m)).astype(np.uint64) + np.uint64(2**63 - 100)
            else:
                vals = np.cumsum(rng.integers(-50, 51, m)).astype(np.int64)
            fl.append((col, pt, vals, None if valid.all() else valid))
            cols[col] = (vals, valid)
        b.add_column_group(sid, ts, fl)
        truth[sid] = [(ts, cols)]
    arena, descs = b.finish()
    return arena, descs, truth


def exact_fit_grid(truth, width, origin, ranges):
    """(first_bucket_start, n_buckets) of the smallest grid holding every row the ranges select (rows outside them may
    fall outside the grid); (0, 1) when nothing is selected."""
    starts = []
    for cgs in truth.values():
        for ts, _ in cgs:
            sel = np.ones(ts.size, dtype=bool)
            if ranges:
                sel = np.zeros(ts.size, dtype=bool)
                for a, b in ranges:
                    sel |= (ts >= a) & (ts <= b)
            t = ts[sel]
            ws, _ = sliding_window(t, width, width, origin)
            with np.errstate(over="ignore"):
                dw = ws - t  # = -(t - origin % w + w) % w, exact
                # rows near the i64 limits whose window start wraps around get no bucket: the scan must report that
                wrapped = ((dw > 0) & (t > np.int64(I64_MAX) - np.maximum(dw, 0))) | \
                          ((dw < 0) & (t < np.int64(I64_MIN) - np.minimum(dw, 0)))
            if (~wrapped).any():
                starts += [int(ws[~wrapped].min()), int(ws[~wrapped].max())]
    if not starts:
        return 0, 1
    lo, hi = min(starts), max(starts)
    nb = (hi - lo) // width + 1
    assert nb < 1 << 22, "sweep grid of %d buckets" % nb
    return lo, nb


def geometry_ranges(kind, t0, step, n, width, origin):
    """The time ranges of one sweep variant (list of closed (a, b))."""
    span = (n - 1) * step
    t_at = lambda k: t0 + (k * step)  # noqa: E731  (row k of block A)
    k1, k2 = n // 5, max(n // 5, (4 * n) // 5)
    clamp = lambda x: min(max(x, I64_MIN), I64_MAX)  # noqa: E731
    if kind == "none":
        return []
    if kind == "rows":
        return [(t_at(k1), t_at(k2))]
    if kind == "inside":
        return [(clamp(t_at(k1) + 1), clamp(t_at(k2) - 1))]
    if kind == "outside":
        return [(clamp(t_at(k1) - 1), clamp(t_at(k2) + 1))]
    if kind == "edges":  # bucket edges +- 1: from one ns after the start of row k1's bucket to one ns past row k2's
        s1, _ = sliding_window(t_at(k1), width, width, origin)
        s2, e2 = sliding_window(t_at(k2), width, width, origin)
        return [(clamp(s1 + 1), clamp(e2))] if s1 + 1 <= clamp(e2) else [(clamp(s1 - 1), clamp(e2 - 1))]
    if kind == "between":  # strictly between two rows of block A (selects rows of blocks B / C at most)
        return [(clamp(t_at(k1) + 1), clamp(t_at(k1 + 1) - 1))] if step >= 2 else [(clamp(t_at(k1) + 1),) * 2]
    if kind == "reversed":  # a > b: selects nothing
        a, b = clamp(t_at(k2)), clamp(t_at(k1) - 1)
        return [(a, b)] if a > b else [(I64_MAX, I64_MIN)]
    if kind == "full":
        return [(I64_MIN, I64_MAX)]
    if kind == "wide":
        return [(clamp(t0 - 3 * span - 5), clamp(t0 + 4 * span + 5))]
    raise ValueError(kind)


def split_ranges(ranges):
    """[a, b] -> [a, m] u [m + 1, b]: the same rows through two ranges (which turns the row-space fast path off)."""
    (a, b), = ranges
    if a >= b:
        return [(a, b), (a, b)]
    m = a + (b - a) // 2
    return [(a, m), (m + 1, b)]


def time_page_is_rle(arena, desc):
    """The DeltaTs kind of a time page (page.rs layout: u32 bitset_len | u64 rows | u32 crc | bitset | data): data[1] >> 4
    is 2 for the run-length form, 1 for simple8b deltas."""
    off = int(desc["offset"])
    bitset_len = int.from_bytes(bytes(arena[off:off + 4]), "big")
    return int(arena[off + 16 + bitset_len + 1]) >> 4 == 2


RANGE_KINDS = ("rows", "inside", "outside", "edges", "between", "reversed", "full", "wide")
ROWS_PER_PAGE = (2, 31, 32, 33, 127, 128, 129, 700, 1, 4097)


def _origin(kind, w, anchor):
    """origin 0, one with origin % w != 0, a negative one, one >= w; `anchor` puts a bucket edge inside the pages."""
    if kind == "zero":
        return 0
    if kind == "mod":
        return wrap64(anchor + max(1, w // 2)) if anchor else (w // 2 + 1 if w > 2 else 1)
    if kind == "neg":
        return -((abs(anchor) % w) + (w + 1) // 3) if w > 1 else -5
    return min(I64_MAX, abs(anchor) % w + 2 * w + 1)  # "big": >= w (saturates for the widest buckets)


def _t0(kind, step, n, origin, w):
    span = (n - 1) * step
    if kind == "pos":
        return 10**12 + 17
    if kind == "straddle":  # rows on both sides of the sign change of t - origin % w + w (truncating % below it)
        om = int(np.fmod(np.int64(origin), np.int64(w)))
        return om - w - (n // 2) * step
    return {"2^62-1": 2**62 - 1, "2^62": 2**62, "-2^62": -2**62, "-2^62-1": -2**62 - 1,
            "max": I64_MAX - span, "min": I64_MIN}[kind]


def geometry_cases():
    """The sweep: (id, step, width, origin, t0, rows per page, range kinds). The step x width product (the widths
    relative to the step), then chosen combinations for constant timestamps and the wide / odd widths."""
    t0_kinds = ("pos", "straddle", "2^62-1", "2^62", "-2^62", "-2^62-1", "max", "min")
    o_kinds = ("zero", "mod", "neg", "big")
    cases = []

    def add(step, w, okind, tkind, n, anchor_row=None):
        k = len(cases)
        span = (n - 1) * step
        if anchor_row is None:
            origin = _origin(okind, w, 0)
            t0 = _t0(tkind, step, n, origin, w)
        else:  # origin relative to the rows: a bucket edge falls on row `anchor_row` + 1/3 step
            t0 = _t0(tkind, step, n, 0, w) if tkind != "straddle" else -(n // 2) * step
            origin = _origin(okind, w, t0 + anchor_row * step + step // 3)
            if tkind == "straddle":
                t0 = _t0(tkind, step, n, origin, w)
        if not (I64_MIN <= t0 and t0 + span <= I64_MAX):
            return
        kinds = ("none", RANGE_KINDS[k % len(RANGE_KINDS)], RANGE_KINDS[(k + 3) % len(RANGE_KINDS)])
        cases.append(("s%d-w%d-o%s-t%s-n%d" % (step, w, okind, tkind, n), step, w, origin, t0, n, kinds))

    for si, d in enumerate((1, 3, 1000, 10**9 + 7, 2**40 + 3)):
        for wi, w in enumerate((6 * d, 6 * d + 1, 6 * d + d // 2, 7 * d - 1, d, d - 1, d // 3)):
            if w <= 0 or (wi in (2,) and d < 2):
                continue
            k = len(cases)
            add(d, w, o_kinds[k % 4], t0_kinds[k % len(t0_kinds)], ROWS_PER_PAGE[k % len(ROWS_PER_PAGE)])
    add(0, 1000, "mod", "pos", 129)                       # constant timestamps: the RLE walk loop
    add(0, 1000, "neg", "straddle", 33)
    add(0, 7, "zero", "max", 31)
    add(1000, 7, "zero", "pos", 129)                      # many empty buckets
    add(1000, 7, "neg", "straddle", 33)
    add(1000, 700_001, "mod", "pos", 700, 350)            # a prime around the page span
    add(1000, 127_031, "neg", "straddle", 128, 60)
    add(1000, 2**16, "zero", "-2^62", 700)                # a power of two
    add(1000, 2**16, "big", "straddle", 129)
    add(1, 2**33 + 5, "mod", "pos", 4097, 2000)           # width / step >= 2^32: q saturates
    add(1, 2**33 + 5, "neg", "2^62-1", 700, 300)
    for w in (2**61 - 1, 2**61, 2**62 + 1, 2**63 - 1):   # the fast path's width limit, magic division l = 61 .. 63
        add(2**40 + 3, w, "mod", "pos", 4097, 2048)
        add(2**40 + 3, w, "neg", "straddle", 700, 350)
        add(10**9 + 7, w, "zero", "max", 129)
        add(10**9 + 7, w, "big", "min", 129)
    add(3, 18, "mod", "2^62", 128)                        # the upper edge of t0 in [-2^62, 2^62)
    add(3, 19, "mod", "-2^62-1", 129)                     # its lower edge
    add(10**9 + 7, 6 * (10**9 + 7) + 1, "big", "max", 700)
    add(10**9 + 7, 6 * (10**9 + 7), "neg", "min", 700)
    return cases


GEOMETRY_CASES = geometry_cases()


def bits_for(x):
    return int(x).bit_length()


def sel_unsupported(query, truth):
    """The scan rejects FIRST / LAST across series when (2 * width, or the selected time span) x slot count does not fit
    its 62-bit tie-break key (TSKV_ERR_UNSUPPORTED)."""
    if not any(c.agg_mask & (cabi.TSKV_AGG_FIRST | cabi.TSKV_AGG_LAST) for c in query.columns):
        return False
    n_slots = len(query.series_ids) if query.series_ids is not None else len(truth)
    slot_bits = 0 if (query.group_by_series or n_slots <= 1) else bits_for(n_slots - 1)
    if slot_bits == 0:
        return False
    if query.width > 0:
        rel = bits_for(2 * query.width) if query.width < 2**61 else 64
    else:
        lo = min(int(ts.min()) for cgs in truth.values() for ts, _ in cgs)
        hi = max(int(ts.max()) for cgs in truth.values() for ts, _ in cgs)
        if query.time_ranges:
            lo = max(lo, min(a for a, _ in query.time_ranges))
            hi = min(hi, max(b for _, b in query.time_ranges))
        rel = 0 if hi < lo else bits_for(hi - lo)
    return rel + slot_bits > 62


def geometry_queries(case, ranges, truth):
    """[(name, query)]: GROUP BY bucket, the same with FIRST / LAST, group_by_series, unbucketed, and one with a predicate
    (so the row keep bits are read). The grid fits the selected rows exactly."""
    _, step, w, origin, t0, n, _ = case
    fbs, nb = exact_fit_grid(truth, w, origin, ranges)
    grid = dict(width=w, origin=origin, first_bucket_start=fbs, n_buckets=nb)
    few = np.array([0, 1, 40, 41, ALL_NULL_SERIES, 80, 81], dtype=np.uint32)  # group_by_series over many buckets
    gbs_ids = few if nb * GEOM_SERIES > 300_000 else None
    pred = [(1, cabi.TSKV_PT_I64, ">=", 0)]
    return [
        ("bucket", make_query(GEOM_FIELDS, GEOM_AGGS, time_ranges=ranges, **grid)),
        ("bucket+sel", make_query(GEOM_FIELDS, ALL_AGGS, time_ranges=ranges, **grid)),
        ("by_series", make_query(GEOM_FIELDS, ALL_AGGS, time_ranges=ranges, group_by_series=True, series_ids=gbs_ids, **grid)),
        ("unbucketed", make_query(GEOM_FIELDS, ALL_AGGS, time_ranges=ranges)),
        ("predicate", make_query(GEOM_FIELDS, GEOM_AGGS, time_ranges=ranges, predicates=pred, **grid)),
    ]
