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
# the kernels. Integer sums are exact Python ints; f64 sums are a class that holds for any summation order starting from
# +0.0 (NaN, an infinity, or finite with an error bound: f64_sum_class). FIRST / LAST follow DESIGN section 7: a run is
# the selected rows of one (slot, column group, bucket) - of one (slot, overlap group, bucket) for merged chunks - and
# only its min-time (max-time) row may contribute, and only with a value; the cell takes the smallest (t, slot) for
# FIRST, the largest t and on a tie the smallest slot for LAST. Tombstones and the overlap merge of chunk files are
# restated here as well (exact_aggregate's `tombstones=` / `files=`).

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


DBL_MAX = float(np.finfo(np.float64).max)
_SCALE = 2.0 ** -64  # magnitudes are compared scaled, so that sums up to 2^1088 stay finite in the reference itself


class OrderDependentSum(ValueError):
    """An f64 cell whose class (finite, +-inf or NaN) depends on the summation order: arenas must not make one."""


def f64_sum_class(x):
    """-> (value, sum|x|) of the f64 SUM of the values x of one cell, the same in every summation order that starts
    from +0.0:
      NaN    if some value is NaN, or the cell holds both +inf and -inf;
      +-inf  if it holds one sign of inf (and the finite values of the other sign cannot overflow), or when its finite
             values all but have one sign and their exact sum is so large that no order stays finite;
      finite otherwise, exactly rounded (math.fsum; +0.0 for a zero sum), when sum|x| (1 + gamma_{n-1}) <= DBL_MAX,
             so that no partial sum of any order overflows (n: the nonzero values). Its error bound comes from sum|x|.
    Raises OrderDependentSum for anything else."""
    x = np.asarray(x, dtype=np.float64)
    if np.isnan(x).any():
        return math.nan, 0.0
    pinf, ninf = bool((x == np.inf).any()), bool((x == -np.inf).any())
    if pinf and ninf:
        return math.nan, 0.0
    f = x[np.isfinite(x)] * _SCALE  # (values below 2^-1010 lose bits here: far too little to move a threshold)
    pos, neg = math.fsum(f[f > 0]), -math.fsum(f[f < 0])
    g = 1 + gamma(max(np.count_nonzero(x) - 1, 0))  # (adding a zero is exact)
    if pinf or ninf:
        if (pos if ninf else neg) * g < DBL_MAX * _SCALE:
            return (math.inf if pinf else -math.inf), 0.0
        raise OrderDependentSum("one sign of inf, and finite values of the other sign that may overflow")
    if (pos + neg) * g <= DBL_MAX * _SCALE:
        s = math.fsum(x)
        return (s if s != 0 else 0.0), math.fsum(np.abs(x))
    s = pos - neg  # any finite result is within gamma_{n-1} (pos + neg) of s: when that is past DBL_MAX, none is finite
    if abs(s) - (g - 1) * (pos + neg) > DBL_MAX * _SCALE and min(pos, neg) * g < DBL_MAX * _SCALE:
        return math.copysign(math.inf, s), 0.0
    raise OrderDependentSum("sum|x| = %g * 2^64 may overflow in some orders" % (pos + neg))


class ExactResult:
    """Expected dense result: values[j, cell] (u64 bits) and validity[j, cell] like ScanResult. For f64 SUM / MEAN
    `center[j]` holds the exactly rounded value (math.fsum) and `bound[j]` the largest error any summation order makes;
    a NaN or infinite center (bound 0) is the class every order gives."""

    def __init__(self, query, n_groups):
        self.names = query.output_names()
        self.n_groups, self.n_buckets = n_groups, query.n_buckets
        n_cells = n_groups * query.n_buckets
        self.values = np.zeros((len(self.names), n_cells), dtype=np.uint64)
        self.validity = np.zeros((len(self.names), n_cells), dtype=bool)
        self.center, self.bound = {}, {}
        self.phys = {c.column_id: c.phys_type for c in query.columns}
        self.exact_sums = {}  # column id -> {cell: (S, n)} of integer columns


def _in_ranges(ts, ranges):
    """Rows of `ts` inside one of the closed ranges (an empty range, a > b, holds none)."""
    m = np.zeros(ts.size, dtype=bool)
    for a, b in ranges:
        m |= (ts >= a) & (ts <= b)
    return m


def tombstone_lists(tombstones):
    """TOMBSTONE_DTYPE array -> (ranges that drop rows of every series, {series: ranges that drop its rows},
    {(series, column): ranges in which the column reads as NULL}). Empty ranges (min > max) are left out."""
    glob, rows, cols = [], {}, {}
    for tb in (tombstones if tombstones is not None else []):
        s, c, a, b = int(tb["series_id"]), int(tb["column_id"]), int(tb["min_ts"]), int(tb["max_ts"])
        if a > b:
            continue
        if s == cabi.TSKV_TOMB_ALL:
            glob.append((a, b))
        elif c == cabi.TSKV_TOMB_ALL:
            rows.setdefault(s, []).append((a, b))
        else:
            cols.setdefault((s, c), []).append((a, b))
    return glob, rows, cols


def _predicates_hold(query, ts, cols):
    """The AND-ed predicates of every row (NULL or an absent column: the comparison is not TRUE)."""
    sel = np.ones(ts.size, dtype=bool)
    for pc, ppt, op, c in query.predicates:
        if pc not in cols:
            sel[:] = False
        else:
            pv, pvalid = cols[pc]
            sel &= np.asarray(pvalid, dtype=bool) & _cmp(ppt, op, pv, c)
    return sel


def overlap_groups(cgs, files):
    """The overlap groups of one series' column groups `cgs` ([(ts, cols)]) with file ids `files` (None: one group per
    column group). A chunk is the column groups of one file, bounded by their min / max time; chunks sorted by (lo, hi,
    file) chain while lo <= the running max hi. -> [[stream, ...]]: a stream per chunk, ordered by file id, each the
    chunk's column group indices by min time."""
    if files is None:
        return [[[k]] for k in range(len(cgs))]
    chunks = {}
    for k, (ts, _) in enumerate(cgs):
        chunks.setdefault(int(files[k]), []).append(k)
    bounds = []
    for f, ks in chunks.items():
        lo = min(int(np.min(cgs[k][0])) for k in ks)
        hi = max(int(np.max(cgs[k][0])) for k in ks)
        bounds.append((lo, hi, f))
    bounds.sort()
    groups, cur, run_max = [], [], None
    for lo, hi, f in bounds:
        if cur and not lo <= run_max:
            groups.append(cur)
            cur = []
        cur.append(f)
        run_max = hi if run_max is None else max(run_max, hi)
    groups.append(cur)
    return [[sorted(chunks[f], key=lambda k: int(np.min(cgs[k][0]))) for f in sorted(g)] for g in groups]


def files_by_series(truth, files):
    """{series: [file id of each of its column groups]} from `files` in truth's order ({} for None)."""
    file_of, k = {}, 0
    if files is not None:
        for sid, cgs in truth.items():
            file_of[sid] = list(files[k:k + len(cgs)])
            k += len(cgs)
        assert k == len(files)
    return file_of


def _merged_rows(cgs, streams, query, qcols, row_drop):
    """The merged rows of one overlap group of two or more chunks: rows of the column groups this scan reads that pass
    the predicates (on their own column group) and no row tombstone; equal times collapse, every query column takes the
    last non-null value in (stream, row) order. -> (times, {column: (values, validity)})."""
    t_all, order_vals = [], {c: ([], []) for c in qcols}
    for stream in streams:
        for k in stream:
            ts, cols = cgs[k]
            if not any(c in cols for c in qcols):
                continue  # a column group without a query column is not read
            ts = np.asarray(ts, dtype=np.int64)
            keep = _predicates_hold(query, ts, cols) & ~_in_ranges(ts, row_drop)
            t_all.append(ts[keep])
            for c in qcols:
                v, valid = cols[c] if c in cols else (np.zeros(ts.size, dtype=np.uint64), np.zeros(ts.size, dtype=bool))
                order_vals[c][0].append(_typed(query_phys(query, c), v)[keep].view(np.uint64))
                order_vals[c][1].append(np.asarray(valid, dtype=bool)[keep])
    t = np.concatenate(t_all) if t_all else np.zeros(0, dtype=np.int64)
    order = np.argsort(t, kind="stable")  # equal times keep their (stream, row) order
    t = t[order]
    starts = np.flatnonzero(np.concatenate([[True], t[1:] != t[:-1]])) if t.size else np.zeros(0, dtype=np.int64)
    out = {}
    for c in qcols:
        v = np.concatenate(order_vals[c][0])[order] if t.size else np.zeros(0, dtype=np.uint64)
        valid = np.concatenate(order_vals[c][1])[order] if t.size else np.zeros(0, dtype=bool)
        if not t.size:
            out[c] = (v, valid)
            continue
        last = np.maximum.reduceat(np.where(valid, np.arange(t.size), -1), starts)
        out[c] = (np.where(last >= 0, v[np.maximum(last, 0)], 0).astype(np.uint64), last >= 0)
    return t[starts] if t.size else t, out


def query_phys(query, column_id):
    return next(c.phys_type for c in query.columns if c.column_id == column_id)


def first_last_rel_bits(truth, query):
    """bits of the time part of the FIRST / LAST tie-break keys: 2 * width when bucketed, else the span of the selected
    times - the query's ranges, tightened on a single-rank scan by the page set's own min / max time."""
    if query.width > 0:
        return bits_for(2 * query.width) if query.width < 2**61 else 64
    lo, hi = I64_MIN, I64_MAX
    if not query.multi_rank:
        lo = min(int(np.min(ts)) for cgs in truth.values() for ts, _ in cgs if len(ts))
        hi = max(int(np.max(ts)) for cgs in truth.values() for ts, _ in cgs if len(ts))
    if query.time_ranges:
        lo = max(lo, min(a for a, _ in query.time_ranges))
        hi = min(hi, max(b for _, b in query.time_ranges))
    return 0 if hi < lo else bits_for(hi - lo)


def exact_aggregate(truth, query, tombstones=None, files=None, key_slots=None):
    """COUNT / SUM / MIN / MAX / MEAN / FIRST / LAST of `query` over `truth` ({series id: [(timestamps, {column id:
    (values, validity)}), ...]}, one entry per column group). A column group that holds none of the query columns is
    never read.
      tombstones  TOMBSTONE_DTYPE array: a row whose time lies in a global or a (series, ALL) range is dropped; a value
                  whose time lies in a (series, column) range reads as NULL.
      files       the file id of every column group, in truth's order (series by series): the chunks of a series that
                  overlap are merged (overlap_groups, _merged_rows), and their merged rows of a bucket form one FIRST /
                  LAST run.
      key_slots   the slot count the tie-break keys are built for (default: the selection's; GROUP BY tags: the whole
                  selection's).
    Raises ReferenceError(TSKV_ERR_UNSUPPORTED) when FIRST / LAST across slots do not fit the 62-bit key, and
    ReferenceError(TSKV_ERR_BUCKET_RANGE) when a selected row (time ranges, predicates, tombstones) has no bucket."""
    slots = [int(s) for s in query.series_ids] if query.series_ids is not None else sorted(truth)
    n_groups = len(slots) if query.group_by_series else 1
    nb = query.n_buckets
    n_cells = n_groups * nb
    qcols = [c.column_id for c in query.columns]
    want_sel = any(c.agg_mask & (cabi.TSKV_AGG_FIRST | cabi.TSKV_AGG_LAST) for c in query.columns)
    n_key = key_slots if key_slots is not None else (len(query.series_ids) if query.series_ids is not None else len(truth))
    slot_bits = 0 if (query.group_by_series or n_key <= 1) else bits_for(n_key - 1)
    if want_sel and slot_bits and first_last_rel_bits(truth, query) + slot_bits > 62:
        raise ReferenceError(cabi.TSKV_ERR_UNSUPPORTED)
    glob, row_tomb, col_tomb = tombstone_lists(tombstones)
    file_of = files_by_series(truth, files)
    units = []  # (slot, times, selected rows, {column: (u64 values, validity)}): one FIRST / LAST run per bucket
    for slot, sid in enumerate(slots):
        cgs = truth.get(sid, [])
        row_drop = glob + row_tomb.get(sid, [])
        for streams in overlap_groups(cgs, file_of.get(sid)):
            if len(streams) >= 2:
                ts, cols = _merged_rows(cgs, streams, query, qcols, row_drop)
                units.append((slot, ts, np.ones(ts.size, dtype=bool), cols))
                continue
            for k in streams[0]:
                ts, cols = cgs[k]
                if not any(c in cols for c in qcols):
                    continue
                ts = np.asarray(ts, dtype=np.int64)
                sel = _predicates_hold(query, ts, cols) & ~_in_ranges(ts, row_drop)
                units.append((slot, ts, sel, {c: (_typed(query_phys(query, c), cols[c][0]).view(np.uint64),
                                                  np.asarray(cols[c][1], dtype=bool)) for c in qcols if c in cols}))
    cells = {c: [] for c in qcols}
    vals = {c: [] for c in qcols}
    firsts = {c: [] for c in qcols}  # (cell, t, slot, value) of every run whose min-time row holds a value
    lasts = {c: [] for c in qcols}
    for slot, ts, sel, cols in units:
        if query.time_ranges:
            sel = sel & _in_ranges(ts, query.time_ranges)
        idx, ok = bucket_index(ts, query)
        if (sel & ~ok).any():
            raise ReferenceError(cabi.TSKV_ERR_BUCKET_RANGE)
        cell = (slot if query.group_by_series else 0) * nb + idx
        rows = np.flatnonzero(sel)
        _, fi = np.unique(idx[rows], return_index=True)  # times ascend: a bucket's first / last selected row
        _, li = np.unique(idx[rows][::-1], return_index=True)
        fr, lr = rows[fi], rows[rows.size - 1 - li]
        for c, (v, valid) in cols.items():
            valid = valid & ~_in_ranges(ts, col_tomb.get((slots[slot], c), []))
            m = sel & valid
            cells[c].append(cell[m])
            vals[c].append(v[m])
            for r, out in ((fr, firsts[c]), (lr, lasts[c])):
                r = r[valid[r]]
                out.append((cell[r], ts[r], np.full(r.size, slot, dtype=np.int64), v[r]))
    sel_out = {}
    for c in qcols:
        for name, cands in (("first", firsts[c]), ("last", lasts[c])):
            cl, t, s, v = (np.concatenate(x) for x in zip(*cands)) if cands else (np.zeros(0, dtype=np.int64),) * 4
            order = np.lexsort((s, t if name == "first" else ~t, cl))
            cl, t, v = cl[order], t[order], np.asarray(v, dtype=np.uint64)[order] if v.size else v.astype(np.uint64)
            head = np.flatnonzero(np.concatenate([[True], cl[1:] != cl[:-1]])) if cl.size else cl
            value, have = np.zeros(n_cells, dtype=np.uint64), np.zeros(n_cells, dtype=bool)
            value[cl[head]], have[cl[head]] = v[head], True
            if not slot_bits:  # keys are the raw times: a FIRST at INT64_MAX / LAST at INT64_MIN is the empty key
                edge = cl[head][t[head] == (I64_MAX if name == "first" else I64_MIN)]
                value[edge], have[edge] = 0, False
            sel_out[(c, name)] = (value, have)
    res = ExactResult(query, n_groups)
    j = 0
    for qc in query.columns:
        c, pt = qc.column_id, qc.phys_type
        cl = np.concatenate(cells[c]) if cells[c] else np.zeros(0, dtype=np.int64)
        v = (np.concatenate(vals[c]) if vals[c] else np.zeros(0, dtype=np.uint64)).view(_typed(pt, []).dtype)
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
                fs[k], ab[k] = f64_sum_class(parts[k])
            n = count.astype(np.float64)
            fin = np.isfinite(fs)
            with np.errstate(invalid="ignore"):
                # fsum is the exactly rounded sum: half an ulp more than gamma_{n-1} for the exact one
                sb = np.where(fin, gamma(np.maximum(n - 1, 0)) * ab * (1 + 2 * _U) + _U * np.abs(fs), 0.0)
                cen_mean = np.where(have, fs / np.maximum(n, 1), 0.0)
            sums = fs.view(np.uint64).copy()
            means = cen_mean.view(np.uint64).copy()
            mb = np.where(fin, sb / np.maximum(n, 1) + 2 * _U * np.abs(np.where(fin, cen_mean, 0.0)), 0.0)
            res_f64 = {"sum": (fs, sb), "mean": (cen_mean, mb)}
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
        out["first"], out["last"] = sel_out[(c, "first")], sel_out[(c, "last")]
        for a in qc.agg_list():
            name = cabi.AGG_NAMES[a]
            if name in out:
                res.values[j], res.validity[j] = out[name]
                if name in res_f64:
                    res.center[j], res.bound[j] = res_f64[name]
            j += 1
    return res


def assert_matches_exact(got, exp, what="", int_mean=True, first_last=True):
    """got: ScanResult; exp: ExactResult. COUNT / integer SUM / MIN / MAX / FIRST / LAST bit-exact (FIRST / LAST
    unless first_last=False), integer MEAN bit-exact (= float(S) / float(n)) unless int_mean=False. f64 SUM / MEAN by
    class (f64_sum_class): a NaN cell must hold some NaN (the payload depends on the order), an inf cell that inf, a
    finite cell a value within the bound, and a zero +0.0."""
    assert got.names == exp.names
    for j, (col, agg) in enumerate(got.names):
        if (agg in ("first", "last") and not first_last) or \
                (agg == "mean" and not int_mean and exp.phys[col] != cabi.TSKV_PT_F64):
            continue
        gv, ev = got.validity[j], exp.validity[j]
        bad = np.nonzero(gv != ev)[0]
        assert bad.size == 0, "%s col %s %s: validity differs at cells %s" % (what, col, agg, bad[:5])
        if j in exp.center:
            cells = np.nonzero(ev)[0]
            g, c, b = got.values[j].view(np.float64)[ev], exp.center[j][ev], exp.bound[j][ev]
            nan, inf = np.isnan(c), np.isinf(c)
            fin = ~(nan | inf)
            with np.errstate(invalid="ignore"):
                ok = np.where(nan, np.isnan(g), np.where(inf, g == c, np.abs(g - c) <= b))
            ok &= ~(fin & (got.values[j][ev] == np.uint64(1 << 63)))  # a zero sum is +0.0
            bad = np.nonzero(~ok)[0]
            assert bad.size == 0, "%s col %s %s at cells %s: got %s, exact %s, bound %s" % (
                what, col, agg, cells[bad[:3]], g[bad[:3]], c[bad[:3]], b[bad[:3]])
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
    return first_last_rel_bits(truth, query) + slot_bits > 62


def raw_key_edge(query, truth):
    """The scan's FIRST / LAST keys are raw row times (group_by_series, or one selected series) and a row lies at
    INT64_MIN or INT64_MAX: there the exact reference keeps the engine's known deviation (DESIGN section 7), which the
    oracle does not have."""
    n_slots = len(query.series_ids) if query.series_ids is not None else len(truth)
    if not (query.group_by_series or n_slots <= 1):
        return False
    return any(((np.asarray(ts) == I64_MIN) | (np.asarray(ts) == I64_MAX)).any() for cgs in truth.values() for ts, _ in cgs)


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


# ---- f64 edge values ---------------------------------------------------------------------------------------------------
# Arenas of f64 pages whose bit patterns reach the rare branches of the Gorilla decoders (meaningful = 64 written as 0,
# leading zeros past the encoder's cap of 31, long runs of repeats, 77-bit elements) and whose values are IEEE special
# values. Every column group holds column 1 (Gorilla) and column 2 (raw: the generic value kernels) with the same rows.
# Four blocks of F64_BLOCK series, by their time pages:
#   A  identical RLE timestamps (whole warps run the uniform bucket schedule);
#   B  RLE timestamps starting sid % 7 rows later (the per-lane segment loop);
#   C  jittered timestamps (simple8b time pages: the fused timestamp + value loop);
#   D  block A's timestamps with the last row moved 2^61 ns later: a raw time page (the generic-time kernels, which read
#      the timestamps from global memory). Bucketed queries leave that row out with a time range.
# The value kind of a series is sid % 10 (F64_KINDS). Rows 127-129 and 255-257 hold the hardest patterns, so that the
# restart points (every 128 rows) and the cuts between page parts land on them.

F64_FIELDS = ((1, cabi.TSKV_PT_F64), (2, cabi.TSKV_PT_F64))
F64_BLOCK = 32
F64_SERIES = 4 * F64_BLOCK
F64_T0, F64_STEP = 10**12 + 17, 1000
F64_LENGTHS = (1, 31, 32, 33, 127, 128, 129, 257, 4097)
F64_KINDS = ("random", "signflip", "bit0_bit63", "runs", "small_xor", "specials", "okey_alone", "okey_mixed", "dbl_max",
             "all_nan")
GORILLA_EOS = 0x7FF80000000000FF  # the Gorilla end-of-stream marker: the encoder refuses it as a value
OKEY_MAX, OKEY_MIN = 0x7FFFFFFFFFFFFFFF, 0xFFFFFFFFFFFFFFFF  # NaNs whose ordered keys are INT64_MAX / INT64_MIN
F64_SPECIALS = np.array([
    0x0000000000000000, 0x8000000000000000,  # +-0.0
    0x7FF0000000000000, 0xFFF0000000000000,  # +-inf
    0x0010000000000000, 0x8010000000000000,  # +-DBL_MIN
    0x0000000000000001, 0x8000000000000001,  # +-2^-1074
    0x000FFFFFFFFFFFFF,                      # the largest subnormal
    0x7FF8000000000000, 0xFFF8000000000000,  # quiet NaNs
    0x7FF0000000000001, 0xFFF4000000000000,  # signalling NaNs
    0x7FF80000000000FE, 0x7FF8000000000100,  # the neighbours of GORILLA_EOS
    OKEY_MAX, OKEY_MIN,
], dtype=np.uint64)
# Finite values are kept below 2^1000 so that no cell's sum|x| comes near DBL_MAX (f64_sum_class): only the dbl_max
# series (+DBL_MAX or -DBL_MAX, one sign per series) overflow, in every order, wherever a cell holds two of their rows.


def _clamp_exp(b):
    """Random bit patterns -> finite values below 2^1000: an exponent field above 2022 loses its top bit."""
    b = np.asarray(b, dtype=np.uint64)
    big = ((b >> np.uint64(52)) & np.uint64(0x7FF)) > 2022
    return np.where(big, b ^ np.uint64(1 << 62), b)


def f64_kind(sid):
    return F64_KINDS[sid % len(F64_KINDS)]


def f64_edge_bits(rng, sid, n):
    """The value bit patterns (uint64) of series `sid` with n rows."""
    kind = f64_kind(sid)
    r = rng.integers(0, 2**64, n, dtype=np.uint64, endpoint=False)
    if kind == "random":
        b = _clamp_exp(r)
    elif kind == "signflip":  # consecutive values differ in bits 63 and 0: leading = 0, meaningful = 64
        odd = (np.arange(n) & 1).astype(np.uint64)
        b = (_clamp_exp(r) & ~np.uint64((1 << 63) | 1)) | (odd << np.uint64(63)) | odd
    elif kind == "bit0_bit63":  # each row flips bit 0, bit 63 or nothing of the row before
        flips = np.array([0, 1, 1 << 63], dtype=np.uint64)[rng.integers(0, 3, n)]
        b = np.bitwise_xor.accumulate(np.concatenate([_clamp_exp(r[:1]), flips[1:]]))
    elif kind == "runs":  # runs of 1 to 300 repeats, then a fresh value
        starts = np.cumsum(rng.integers(1, 301, n))
        b = _clamp_exp(r)[np.searchsorted(starts, np.arange(n), side="right")]
    elif kind == "small_xor":  # XORs below 2^32: 32 to 63 leading zeros (past the cap of 31)
        x = r >> np.uint64(32)
        x >>= rng.integers(0, 32, n).astype(np.uint64)
        b = np.bitwise_xor.accumulate(np.concatenate([_clamp_exp(r[:1]), x[1:]]))
    elif kind == "specials":
        norm = rng.normal(0, 1e3, n).view(np.uint64)
        b = np.where(rng.random(n) < 0.6, F64_SPECIALS[rng.integers(0, F64_SPECIALS.size, n)], norm)
        if sid % 20 == 5:
            b[0] = 0xFFF8000000000000  # a NaN at the first row: FIRST must return it
    elif kind == "okey_alone":
        b = np.full(n, OKEY_MAX if sid % 20 == 6 else OKEY_MIN, dtype=np.uint64)
    elif kind == "okey_mixed":
        b = _clamp_exp(r)
        b[rng.random(n) < 0.05] = OKEY_MAX if sid % 20 == 7 else OKEY_MIN
        b[rng.random(n) < 0.02] = OKEY_MIN if sid % 20 == 7 else OKEY_MAX
    elif kind == "dbl_max":
        b = np.full(n, 0x7FEFFFFFFFFFFFFF | ((sid // 10 % 2) << 63), dtype=np.uint64)
    else:  # all_nan
        b = F64_SPECIALS[9:17][rng.integers(0, 8, n)]  # NaNs of both signs and several payloads
    if kind in ("random", "signflip", "bit0_bit63", "runs", "small_xor", "okey_mixed", "specials"):
        # the hardest transitions around rows 128 and 256: a 77-bit element (meaningful 64), an XOR of one bit
        # (leading 63), a repeat, and for the specials a NaN, -inf and the INT64_MAX key
        for r0 in (127, 255):
            if n > r0 + 2:
                if kind == "specials":
                    b[r0:r0 + 3] = [OKEY_MIN, 0xFFF0000000000000, OKEY_MAX]
                else:
                    h = int(b[r0 - 1]) ^ 0x8000000000000001
                    b[r0:r0 + 3] = [h, h ^ 1, h ^ 1]
    assert not (b == GORILLA_EOS).any()
    return b


def f64_finite_series(ids):
    """The series of `ids` whose values are all finite and below 2^1000 (their sums are finite in every cell)."""
    return np.array([s for s in ids if f64_kind(s) in ("random", "signflip", "bit0_bit63", "runs", "small_xor")],
                    dtype=np.uint32)


def f64_edge_timestamps(rng, sid, n):
    blk = sid // F64_BLOCK
    k = np.arange(n, dtype=np.int64)
    if blk == 1:
        start = sid % 7 if n > 14 else 0
        k = k[: n - start] + start
    ts = F64_T0 + k * F64_STEP
    if blk == 2 and n > 2:
        jit = rng.integers(0, F64_STEP, n)
        jit[0] = jit[-1] = 0
        ts = ts + jit
    if blk == 3 and n > 1:
        ts[-1] = F64_T0 + 2**61  # a delta past 2^60: the writer falls back to a raw time page
    return ts


def f64_edge_arena(seed, n, ids=range(F64_SERIES)):
    """-> (arena, descs, truth) of f64 edge pages of n rows (block B: fewer) for the series `ids`; series 3, 10, 17, ...
    hold nulls."""
    rng = np.random.default_rng(seed)
    b = datagen.ArenaBuilder()
    truth = {}
    for sid in ids:
        ts = f64_edge_timestamps(rng, sid, n)
        m = ts.size
        bits = f64_edge_bits(rng, sid, m)
        valid = rng.random(m) >= 0.25 if sid % 7 == 3 else np.ones(m, dtype=bool)
        vals = bits.view(np.float64)
        vv = None if valid.all() else valid
        b.add_column_group(sid, ts, [(1, cabi.TSKV_PT_F64, vals, vv), (2, cabi.TSKV_PT_F64, vals, vv, datagen.encode_raw)])
        truth[sid] = [(ts, {1: (vals, valid), 2: (vals, valid)})]
    arena, descs = b.finish()
    return arena, descs, truth


def f64_edge_queries(n, ids=range(F64_SERIES)):
    """[(name, query, extra)]: extra = {} or {"group_ids": ..., "n_groups": ...} (GROUP BY tags) or {"slide": ...}."""
    w = F64_STEP * max(1, n // 5)
    fbs, nb = bucket_spec(F64_T0, F64_T0 + n * F64_STEP, w)
    grid = dict(width=w, first_bucket_start=fbs, n_buckets=nb, time_ranges=[(F64_T0, F64_T0 + n * F64_STEP)])
    aggs = ("count", "sum", "min", "max", "mean")
    mixed = np.array([s for s in ids if f64_kind(s) != "dbl_max"], dtype=np.uint32)  # (two signs of DBL_MAX in a cell
    finite = f64_finite_series(ids)                                                   # may or may not overflow)
    k = 3
    sgrid = dict(width=k * w, first_bucket_start=fbs - (k - 1) * w, n_buckets=nb + k - 1,
                 time_ranges=grid["time_ranges"])
    return [
        ("bucket", make_query(F64_FIELDS, aggs, series_ids=mixed, **grid), {}),
        ("bucket+sel", make_query(F64_FIELDS, ALL_AGGS, series_ids=mixed, **grid), {}),
        ("bucket_finite", make_query(F64_FIELDS, aggs, series_ids=finite, **grid), {}),
        ("by_series", make_query(F64_FIELDS, ALL_AGGS, group_by_series=True, **grid), {}),
        ("unbucketed", make_query(F64_FIELDS, aggs, series_ids=mixed), {}),
        ("tags", make_query(F64_FIELDS, aggs, series_ids=mixed, **grid),
         {"group_ids": (mixed % 5).astype(np.uint32), "n_groups": 5}),
        ("sliding", make_query(F64_FIELDS, aggs, series_ids=mixed, **sgrid), {"slide": w}),
    ]


def f64_edge_expected(truth, query, extra):
    """The exact reference of one f64_edge_queries entry."""
    from tests.group_reference import exact_aggregate_grouped
    from tests.sliding_reference import expand_aggregate
    if "group_ids" in extra:
        return exact_aggregate_grouped(truth, query, extra["group_ids"], extra["n_groups"])
    if "slide" in extra:
        return expand_aggregate(truth, query, extra["slide"])
    return exact_aggregate(truth, query)
