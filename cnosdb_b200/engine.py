"""Host-side mirror of the reference's reader interface for the scan path, over the C ABI.

Reference seam (paths relative to the reference tree):
  QueryOption / time ranges / aggregates   tskv/src/reader/iterator.rs:713-741
  BatchReader::process                      tskv/src/reader/mod.rs:159-164
  TsmReader::read_adjacent_pages + CRC      tskv/src/tsm/reader.rs:236-264
  Page::to_arrow_array                      tskv/src/tsm/page.rs:96-98
This module only marshals arguments: all compute happens in libtskv_gpu.so (CUDA, sm_90a).
"""
import ctypes as C

import numpy as np

from . import cabi
from .cabi import (TSKV_AGG_COUNT, TSKV_AGG_FIRST, TSKV_AGG_LAST, TSKV_AGG_M2, TSKV_AGG_MAX, TSKV_AGG_MEAN,
                   TSKV_AGG_MIN, TSKV_AGG_SUM, TSKV_PT_F64, TSKV_PT_I64, TSKV_PT_TIME, TSKV_PT_U64)

AGG_BITS = {"count": TSKV_AGG_COUNT, "sum": TSKV_AGG_SUM, "min": TSKV_AGG_MIN, "max": TSKV_AGG_MAX,
            "mean": TSKV_AGG_MEAN, "avg": TSKV_AGG_MEAN, "first": TSKV_AGG_FIRST, "last": TSKV_AGG_LAST,
            "m2": TSKV_AGG_M2}
# DataFusion's statistical aggregates, computed on the host from the scan's COUNT and M2 (sum of squared deviations):
# name -> (divisor n - ddof, sqrt?). stddev / var are the sample forms.
STAT_AGGS = {"var": (1, False), "var_samp": (1, False), "var_pop": (0, False),
             "stddev": (1, True), "stddev_samp": (1, True), "stddev_pop": (0, True)}


def stat_from_m2(name, count, m2, valid):
    """DataFusion's final formula of a STAT_AGGS aggregate from COUNT and M2 cells (numpy arrays): var_pop = m2 / n,
    var_samp = m2 / (n - 1), stddev* = sqrt(var*). Returns (values f64, validity): NULL where n <= ddof (an empty cell; a
    one-value cell for the sample forms)."""
    ddof, root = STAT_AGGS[name]
    n = np.asarray(count, dtype=np.uint64).astype(np.float64)
    ok = np.asarray(valid, dtype=bool) & (n > ddof)
    with np.errstate(divide="ignore", invalid="ignore"):
        v = np.where(ok, np.asarray(m2, dtype=np.float64) / np.where(ok, n - ddof, 1.0), 0.0)
    if root:
        with np.errstate(invalid="ignore"):
            v = np.sqrt(v)
    return v, ok


# DataFusion's covariance / correlation, computed on the host from a column pair's n and co-moments (QueryOption.pairs).
PAIR_AGGS = ("covar", "covar_samp", "covar_pop", "corr")
PAIR_RAW = ("n", "c", "m2x", "m2y")


def pair_stat(name, n, c, m2x, m2y, valid):
    """DataFusion's final formula of a PAIR_AGGS aggregate from a pair's cells (numpy arrays): covar = covar_samp =
    C / (n - 1), covar_pop = C / n, corr = (C / n) / sqrt(M2x / n) / sqrt(M2y / n) in that order, 0.0 when either root is
    0. Returns (values f64, validity): NULL where n == 0, and for the sample form where n == 1."""
    n = np.asarray(n, dtype=np.uint64).astype(np.float64)
    ok = np.asarray(valid, dtype=bool) & (n > (1 if name in ("covar", "covar_samp") else 0))
    c, m2x, m2y = (np.asarray(a, dtype=np.float64) for a in (c, m2x, m2y))
    d = np.where(ok, n, 1.0)
    with np.errstate(divide="ignore", invalid="ignore"):
        if name in ("covar", "covar_samp"):
            v = c / np.where(ok, n - 1.0, 1.0)
        elif name == "covar_pop":
            v = c / d
        else:
            s1, s2 = np.sqrt(m2x / d), np.sqrt(m2y / d)
            v = np.where((s1 == 0.0) | (s2 == 0.0), 0.0, (c / d) / s1 / s2)
    return np.where(ok, v, 0.0), ok


def _wrap64(x):
    x &= (1 << 64) - 1
    return x - (1 << 64) if x >> 63 else x


def _cmod(a, b):
    """a % b with the sign of a (C / Rust `%`)."""
    r = abs(a) % abs(b)
    return -r if a < 0 else r


def window_last_start(t, window, slide, origin):
    """Start of the last window holding t: t - ((t - origin % window) + slide) % slide, with truncating `%` and wrapping
    i64 arithmetic like the reference's window expression (transform_time_window.rs:251-296)."""
    return _wrap64(t - _cmod(_wrap64(_wrap64(t - _cmod(origin, window)) + slide), slide))


def sliding_window_grid(lo, hi, window, slide, origin=0):
    """(first_bucket_start, n_buckets) of the windows of time_window(time, window, slide, origin) that hold the rows of
    the closed range [lo, hi]: from the first window of lo, last_start(lo) - (k - 1) * slide with k = ceil(window /
    slide), to the last window of hi, last_start(hi). For rows whose dividend t - origin % window + slide is >= 0 and
    does not wrap (the reference's floor regime)."""
    k = -(-window // slide)
    first = window_last_start(lo, window, slide, origin) - (k - 1) * slide
    last = window_last_start(hi, window, slide, origin)
    return first, (last - first) // slide + 1


_PER_SECOND = {"s": 1, "ms": 1_000, "us": 1_000_000, "ns": 1_000_000_000}
_FIXED_DAYS = {"week": 7, "day": 1}
_FIXED_SECONDS = {"hour": 3600, "minute": 60, "second": 1}
CALENDAR_UNITS = ("year", "quarter", "month", "week", "day", "hour", "minute", "second")


def _days_from_civil(y, m, d):
    """Days since 1970-01-01 of the proleptic Gregorian date y-m-d (any year)."""
    y -= m <= 2
    era = y // 400
    yoe = y - era * 400
    doy = (153 * (m + (-3 if m > 2 else 9)) + 2) // 5 + d - 1
    doe = yoe * 365 + yoe // 4 - yoe // 100 + doy
    return era * 146097 + doe - 719468


def _civil_from_days(z):
    """(year, month, day) of the proleptic Gregorian date `z` days after 1970-01-01 (z may be negative)."""
    z += 719468
    era = z // 146097
    doe = z - era * 146097
    yoe = (doe - doe // 1460 + doe // 36524 - doe // 146096) // 365
    doy = doe - (365 * yoe + yoe // 4 - yoe // 100)
    mp = (5 * doy + 2) // 153
    d = doy - (153 * mp + 2) // 5 + 1
    m = mp + (3 if mp < 10 else -9)
    return yoe + era * 400 + (m <= 2), m, d


def calendar_edges(unit, t_lo, t_hi, precision="ns"):
    """Time-bucket edges of GROUP BY date_trunc(unit, time) over the rows of [t_lo, t_hi] (int64 timestamps in
    `precision`: "s", "ms", "us" or "ns"): an int64 array from date_trunc(unit, t_lo) to the first unit start after
    t_hi, for Engine.scan_aggregate(..., edges=...). Proleptic Gregorian calendar in UTC (the time column carries no
    zone), times before 1970 floor to the unit start at or before them, weeks start on Monday."""
    if unit not in CALENDAR_UNITS:
        raise ValueError("calendar_edges: unit must be one of %s" % (CALENDAR_UNITS,))
    if precision not in _PER_SECOND:
        raise ValueError("calendar_edges: precision must be one of %s" % (tuple(_PER_SECOND),))
    t_lo, t_hi = int(t_lo), int(t_hi)
    if t_lo > t_hi:
        raise ValueError("calendar_edges: t_lo > t_hi")
    per_day = 86400 * _PER_SECOND[precision]
    if unit in _FIXED_SECONDS or unit in _FIXED_DAYS:
        if unit in _FIXED_SECONDS:
            w, start = _FIXED_SECONDS[unit] * _PER_SECOND[precision], 0
        else:  # weeks from Monday 1969-12-29 (1970-01-01 is a Thursday)
            w, start = _FIXED_DAYS[unit] * per_day, -3 * per_day if unit == "week" else 0
        first = start + (t_lo - start) // w * w
        n = (t_hi - first) // w + 1
        edges = [first + k * w for k in range(n + 1)]
    else:
        months = {"year": 12, "quarter": 3, "month": 1}[unit]
        y, m, _ = _civil_from_days(t_lo // per_day)
        k = (y * 12 + m - 1) // months * months  # months since year 0 of the unit's start
        edges = []
        while True:
            e = _days_from_civil(k // 12, k % 12 + 1, 1) * per_day
            edges.append(e)
            if e > t_hi:
                break
            k += months
    if edges[0] < -2**63 or edges[-1] >= 2**63:
        raise ValueError("calendar_edges: the edges leave the int64 range")
    return np.array(edges, dtype=np.int64)


# date_part units calendar_parts supports: the date_trunc unit whose periods its edges follow, and the values of the
# cyclic units (output bucket j holds the rows whose part is values[j]; year: the years present)
PART_UNITS = {"year": ("year", None), "quarter": ("quarter", range(1, 5)), "month": ("month", range(1, 13)),
              "week": ("week", range(1, 54)), "day": ("day", range(1, 32)), "doy": ("day", range(1, 367)),
              "dow": ("day", range(0, 7)), "hour": ("hour", range(0, 24)), "minute": ("minute", range(0, 60))}


def _iso_week(days):
    """ISO 8601 week number of the Monday `days` days after 1970-01-01: the week of its Thursday, counted in the
    Thursday's year (week 1 holds the year's first Thursday)."""
    thu = days + 3
    y, _, _ = _civil_from_days(thu)
    return (thu - _days_from_civil(y, 1, 1)) // 7 + 1


def calendar_parts(unit, t_lo, t_hi, precision="ns"):
    """Labelled time buckets of GROUP BY date_part(unit, time) / EXTRACT(unit FROM time) over the rows of [t_lo, t_hi]:
    (edges, labels, part_values) for Engine.scan_aggregate(..., edges=edges, labels=labels) with query.n_buckets =
    len(part_values). edges are calendar_edges of the unit's periods (date_trunc('day') edges for day, doy and dow),
    labels[b] is the output bucket of period b, and output bucket j holds the rows whose date_part(unit, time) equals
    part_values[j] (float64, as date_part returns). Units: year (the years present), quarter 1-4, month 1-12, week (ISO
    8601 week number 1-53: weeks start on Monday and belong to the year of their Thursday), day (of the month, 1-31), doy
    (1-366), dow (0 = Sunday .. 6), hour 0-23 and minute 0-59. Proleptic Gregorian calendar in UTC, floor semantics
    before 1970. second and finer units and epoch are refused: their parts are fractional, not a small set of groups."""
    if unit not in PART_UNITS:
        raise ValueError("calendar_parts: unit must be one of %s" % (tuple(PART_UNITS),))
    period, values = PART_UNITS[unit]
    edges = calendar_edges(period, t_lo, t_hi, precision)
    starts = [int(e) for e in edges[:-1]]
    per_day = 86400 * _PER_SECOND[precision]
    if unit == "year":
        values = [_civil_from_days(s // per_day)[0] for s in starts]
        part = values
    elif unit in ("hour", "minute"):
        w = _FIXED_SECONDS[unit] * _PER_SECOND[precision]
        part = [s // w % len(values) for s in starts]
    elif unit == "week":
        part = [_iso_week(s // per_day) for s in starts]
    else:
        part = []
        for s in starts:
            days = s // per_day
            y, m, d = _civil_from_days(days)
            part.append({"quarter": (m - 1) // 3 + 1, "month": m, "day": d, "doy": days - _days_from_civil(y, 1, 1) + 1,
                         "dow": (days + 4) % 7}[unit])  # (1970-01-01 was a Thursday)
    values = list(values)
    index = {v: j for j, v in enumerate(values)}
    labels = np.array([index[p] for p in part], dtype=np.uint32)
    return edges, labels, np.array(values, dtype=np.float64)


class TskvError(RuntimeError):
    """Mirrors TskvError::Decode / TsmPageFileHashCheckFailed: carries the status code."""

    def __init__(self, status, message, page=-1):
        super().__init__("%s (status %d = %s, page %d)" % (
            message, status, cabi.STATUS_NAMES.get(status, "?"), page))
        self.status = status
        self.page = page


class PushedAggregate:
    """One projected value column with its aggregate set (extends PushedAggregateFunction::Count). "median" has no mask
    bit: it makes the column a median operand (after the pairs' operands, agg_mask 0), and a column that asks for nothing
    else has no projected entry. "increase" (increase(time, x ORDER BY time)) likewise makes it an increase operand, after
    the medians' operands."""

    def __init__(self, column_id, phys_type, aggs):
        self.column_id = int(column_id)
        self.phys_type = int(phys_type)
        self.median = False
        self.increase = False
        if isinstance(aggs, int):
            self.agg_mask = aggs
        else:
            self.agg_mask = 0
            for a in aggs:
                if a == "median":
                    self.median = True
                    continue
                if a == "increase":
                    self.increase = True
                    continue
                # var* / stddev* ask the scan for COUNT | M2; ScanResult.column derives them
                self.agg_mask |= (TSKV_AGG_COUNT | TSKV_AGG_M2) if a in STAT_AGGS else AGG_BITS[a]

    def agg_list(self):
        return [b for b in (1, 2, 4, 8, 16, 32, 64, 128) if self.agg_mask & b]


class QueryOption:
    """The pushed-down scan: series selection, closed time ranges, bucket expression, aggregates."""

    def __init__(self, columns, series_ids=None, time_ranges=(), origin=0, width=0,
                 first_bucket_start=0, n_buckets=1, group_by_series=False, multi_rank=False, predicates=(), pairs=()):
        self.columns = list(columns)
        # column pairs (covar* / corr): (x_id, x_phys_type, y_id, y_phys_type); ScanResult.pair reads them
        self.pairs = [(int(a), int(b), int(c), int(d)) for a, b, c, d in pairs]
        self.series_ids = None if series_ids is None else np.ascontiguousarray(series_ids, dtype=np.uint32)
        self.time_ranges = [(int(a), int(b)) for a, b in time_ranges]
        self.origin = int(origin)
        self.width = int(width)
        self.first_bucket_start = int(first_bucket_start)
        self.n_buckets = int(n_buckets)
        self.group_by_series = bool(group_by_series)
        # field comparisons AND-ed into the row filter: (column_id, phys_type, op, constant), op in == != < <= > >=
        self.predicates = [(int(c), int(pt), op if isinstance(op, int) else cabi.CMP_OPS[op], v) for c, pt, op, v in predicates]
        self.multi_rank = bool(multi_rank)  # TSKV_QUERY_MULTI_RANK: partials get merged with other ranks'
        self._keep = None

    def to_c(self):
        q = cabi.Query()
        if self.series_ids is not None:
            q.series_ids = self.series_ids.ctypes.data_as(C.POINTER(C.c_uint32))
            q.n_series = len(self.series_ids)
        tr = (cabi.TimeRange * max(1, len(self.time_ranges)))()
        for i, (a, b) in enumerate(self.time_ranges):
            tr[i].min_ts, tr[i].max_ts = a, b
        q.time_ranges = tr
        q.n_time_ranges = len(self.time_ranges)
        q.origin, q.width = self.origin, self.width
        q.first_bucket_start, q.n_buckets = self.first_bucket_start, self.n_buckets
        q.group_by_series = 1 if self.group_by_series else 0
        proj = self.projected()
        meds = [(c.column_id, c.phys_type) for c in self.columns if getattr(c, "median", False)]
        incs = [(c.column_id, c.phys_type) for c in self.columns if getattr(c, "increase", False)]
        q.reserved = ((cabi.TSKV_QUERY_MULTI_RANK if self.multi_rank else 0) | cabi.query_medians(len(meds)) |
                      cabi.query_increases(len(incs)))
        ops = [o for x, xt, y, yt in self.pairs for o in ((x, xt), (y, yt))] + meds + incs
        cols = (cabi.AggColumn * max(1, len(proj) + len(ops)))()
        for i, c in enumerate(proj):
            cols[i].column_id, cols[i].phys_type, cols[i].agg_mask = c.column_id, c.phys_type, c.agg_mask
        for i, (cid, pt) in enumerate(ops):  # the pairs', medians' and increases' operands follow the projected columns
            cols[len(proj) + i].column_id, cols[len(proj) + i].phys_type = cid, pt
        q.columns = cols
        q.n_columns = len(proj)
        q.n_pairs = len(self.pairs)
        preds = (cabi.FieldPredicate * max(1, len(self.predicates)))()
        for i, (c, pt, op, v) in enumerate(self.predicates):
            preds[i].column_id, preds[i].phys_type, preds[i].op = c, pt, op
            if pt == TSKV_PT_F64:
                preds[i].value = int(np.float64(v).view(np.uint64))
            else:
                preds[i].value = int(v) & 0xFFFFFFFFFFFFFFFF
        if self.predicates:
            q.predicates = preds
            q.n_predicates = len(self.predicates)
        self._keep = (tr, cols, preds)  # keep the ctypes arrays alive as long as the query
        return q

    def projected(self):
        """The columns with a projected entry (an aggregate other than median and increase)."""
        return [c for c in self.columns if c.agg_mask or not (getattr(c, "median", False) or getattr(c, "increase", False))]

    def output_names(self):
        return ([(c.column_id, cabi.AGG_NAMES[a]) for c in self.projected() for a in c.agg_list()] +
                [(("pair", k), r) for k in range(len(self.pairs)) for r in PAIR_RAW] +
                [(c.column_id, "median") for c in self.columns if getattr(c, "median", False)] +
                [(c.column_id, "increase") for c in self.columns if getattr(c, "increase", False)])


class ScanResult:
    """Dense result: values[j, cell] (u64 bit patterns) + validity[j, cell] (bool)."""

    def __init__(self, query, layout, values, bitmaps):
        self.names = query.output_names()
        self.n_groups = int(layout.n_groups)
        self.n_buckets = query.n_buckets
        self.values = values.reshape(int(layout.n_out), int(layout.n_cells))
        bits = np.unpackbits(bitmaps.reshape(int(layout.n_out), int(layout.bitmap_stride)), axis=1,
                             bitorder="little")
        self.validity = bits[:, : int(layout.n_cells)].astype(bool)
        self.phys = {(c.column_id): c.phys_type for c in query.columns}

    def pair(self, k, name):
        """(values f64 / u64 for n, validity) of column pair k, shaped [n_groups, n_buckets]: one of PAIR_AGGS (covar,
        covar_samp, covar_pop, corr), derived on the host by pair_stat, or the raw n / c / m2x / m2y."""
        def raw(r):
            j = self.names.index((("pair", k), r))
            v = self.values[j].view(np.uint64 if r == "n" else np.float64)
            shape = (self.n_groups, self.n_buckets)
            return v.reshape(shape), self.validity[j].reshape(shape)
        if name in PAIR_RAW:
            return raw(name)
        n, _ = raw("n")
        (c, ok), (m2x, _), (m2y, _) = raw("c"), raw("m2x"), raw("m2y")
        return pair_stat(name, n, c, m2x, m2y, ok)

    def column(self, column_id, agg):
        """(typed values, validity) of one output column, shaped [n_groups, n_buckets]. agg may also name one of STAT_AGGS
        (var, var_samp, var_pop, stddev, stddev_samp, stddev_pop), derived from the column's count and m2, or "median" /
        "increase" (the operand's type)."""
        if agg in STAT_AGGS:
            n, _ = self.column(column_id, "count")
            m2, ok = self.column(column_id, "m2")
            return stat_from_m2(agg, n, m2, ok)
        j = self.names.index((column_id, agg))
        raw = self.values[j]
        pt = self.phys[column_id]
        if agg == "count":
            v = raw.view(np.uint64)
        elif agg in ("mean", "m2") or pt == TSKV_PT_F64:
            v = raw.view(np.float64)
        elif pt == TSKV_PT_I64:
            v = raw.view(np.int64)
        else:
            v = raw.view(np.uint64)
        return (v.reshape(self.n_groups, self.n_buckets),
                self.validity[j].reshape(self.n_groups, self.n_buckets))


class PageSet:
    """Device-resident page arena + descriptor tables (the engine's view of cached TsmReaders)."""

    def __init__(self, engine, handle, n_pages):
        self.engine = engine
        self.handle = handle
        self.n_pages = n_pages

    def set_tombstones(self, tombs):
        """Attach the TsmTombstone ranges (cabi.TOMBSTONE_DTYPE array or cabi.tombstones([...]) input);
        replaces the previous set, an empty one clears it. Applies to every later scan of this page set."""
        if not isinstance(tombs, np.ndarray):
            tombs = cabi.tombstones(list(tombs))
        tombs = np.ascontiguousarray(tombs, dtype=cabi.TOMBSTONE_DTYPE)
        self.engine._check(self.engine.lib.tskvgpu_pages_set_tombstones(
            self.engine.ctx, self.handle, tombs.ctypes.data if len(tombs) else None, len(tombs)))

    def set_chunk_files(self, cg_file_ids):
        """File id of every column group (descriptor order): later scans merge + de-duplicate the chunks of a series
        whose time ranges overlap (DataMerger semantics: rows with equal time collapse, the newest file's non-null value
        wins per column). An empty list clears."""
        ids = np.ascontiguousarray(cg_file_ids, dtype=np.uint64)
        self.engine._check(self.engine.lib.tskvgpu_pages_set_chunk_files(
            self.engine.ctx, self.handle, ids.ctypes.data if len(ids) else None, len(ids)))

    def set_value_stats(self, stats):
        """PageMeta.statistics per descriptor (cabi.VALUE_STATS_DTYPE: min / max bit patterns + TSKV_STATS_MINMAX): scans
        with field predicates skip the column groups the bounds rule out, also on host-resident page sets."""
        st = np.ascontiguousarray(stats, dtype=cabi.VALUE_STATS_DTYPE)
        self.engine._check(self.engine.lib.tskvgpu_pages_set_value_stats(self.engine.ctx, self.handle, st.ctypes.data, len(st)))

    def set_time_bounds(self, bounds):
        """Per-column-group (min_ts, max_ts), ColumnGroup::time_range() order = descriptor order: lets scans with time
        ranges skip whole column groups (statistics pruning). bounds: [(lo, hi), ...] or an int64 array of shape [n, 2]."""
        b = np.ascontiguousarray(bounds, dtype=np.int64).reshape(-1, 2)
        self.engine._check(self.engine.lib.tskvgpu_pages_set_time_bounds(self.engine.ctx, self.handle, b.ctypes.data, len(b)))

    def close(self):
        if self.handle and self.engine.ctx:
            self.engine.lib.tskvgpu_pages_destroy(self.engine.ctx, self.handle)
        self.handle = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


class PreparedScan:
    def __init__(self, engine, pages, query, handle, layout):
        self.engine, self.pages, self.query, self.handle, self.layout = engine, pages, query, handle, layout

    def run(self):
        self.engine._check(self.engine.lib.tskvgpu_scan_run(self.engine.ctx, self.handle))

    def enqueue(self):
        """Launches one full pass on the engine stream without synchronising the host."""
        self.engine._check(self.engine.lib.tskvgpu_scan_enqueue(self.engine.ctx, self.handle))

    def sync(self):
        self.engine._check(self.engine.lib.tskvgpu_scan_sync(self.engine.ctx, self.handle))

    def partials(self):
        v = cabi.PartialsView()
        self.engine._check(self.engine.lib.tskvgpu_scan_partials(self.engine.ctx, self.handle, C.byref(v)))
        return v

    def work_list(self):
        """The work list of the last pass (tskvgpu_scan_work_list): dict of region_start, fill, work_page, work_slot,
        work_qcol and the page set's per-descriptor page_bin / page_narrow."""
        lib, ctx = self.engine.lib, self.engine.ctx
        nb, ni = C.c_uint32(0), C.c_uint32(0)
        self.engine._check(lib.tskvgpu_scan_work_list(ctx, self.handle, C.byref(nb), C.byref(ni), *([None] * 7)))
        n_descs = self.pages.n_pages
        out = {"region_start": np.zeros(nb.value + 1, np.uint32), "fill": np.zeros(nb.value, np.uint32),
               "work_page": np.zeros(ni.value, np.uint32), "work_slot": np.zeros(ni.value, np.uint32),
               "work_qcol": np.zeros(ni.value, np.uint8), "page_bin": np.zeros(n_descs, np.uint8),
               "page_narrow": np.zeros(n_descs, np.uint8)}
        self.engine._check(lib.tskvgpu_scan_work_list(ctx, self.handle, C.byref(nb), C.byref(ni),
                                                      *[a.ctypes.data for a in out.values()]))
        return out

    def exchange_view(self):
        """(device pointer, length in 8-byte words) of the region a multi-GPU run all-gathers."""
        a, b = C.c_uint64(0), C.c_uint64(0)
        self.engine._check(self.engine.lib.tskvgpu_scan_exchange_view(self.engine.ctx, self.handle, C.byref(a), C.byref(b)))
        return a.value, b.value

    def exchange(self):
        """The multi-GPU exchange inside the library: one ncclAllGather of the exchange region + the local merge
        (Engine.comm_init first)."""
        self.engine._check(self.engine.lib.tskvgpu_scan_exchange(self.engine.ctx, self.handle))

    def merge_gathered(self, gathered_ptr, n_ranks):
        self.engine._check(self.engine.lib.tskvgpu_scan_merge_gathered(self.engine.ctx, self.handle, gathered_ptr, n_ranks))

    def snapshot_keys(self):
        self.engine._check(self.engine.lib.tskvgpu_scan_snapshot_keys(self.engine.ctx, self.handle))

    def mask_values(self):
        self.engine._check(self.engine.lib.tskvgpu_scan_mask_values(self.engine.ctx, self.handle))

    def finalize(self):
        L = self.layout
        values = np.empty(int(L.n_out * L.n_cells), dtype=np.uint64)
        bitmaps = np.empty(int(L.validity_bytes), dtype=np.uint8)
        self.engine._check(self.engine.lib.tskvgpu_scan_finalize(
            self.engine.ctx, self.handle, values.ctypes.data, bitmaps.ctypes.data))
        return ScanResult(self.query, L, values, bitmaps)

    def finalize_device(self):
        a, b = C.c_uint64(0), C.c_uint64(0)
        self.engine._check(self.engine.lib.tskvgpu_scan_finalize_device(
            self.engine.ctx, self.handle, C.byref(a), C.byref(b)))
        return a.value, b.value

    def close(self):
        if self.handle and self.engine.ctx:  # (an engine closed first has already released the device)
            self.engine.lib.tskvgpu_scan_destroy(self.engine.ctx, self.handle)
        self.handle = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


class Engine:
    """One CUDA device + stream (tskv_ctx)."""

    def __init__(self, device=0):
        self.lib = cabi.load_gpu_library()
        ctx = C.c_void_p()
        st = self.lib.tskvgpu_ctx_create(int(device), C.byref(ctx))
        if st != cabi.TSKV_OK:
            raise TskvError(st, "tskvgpu_ctx_create(device=%d) failed: no usable CUDA device" % device)
        self.ctx = ctx
        self.device = int(device)

    def close(self):
        if self.ctx:
            self.lib.tskvgpu_ctx_destroy(self.ctx)
            self.ctx = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def _check(self, st):
        if st != cabi.TSKV_OK:
            msg = self.lib.tskvgpu_last_error(self.ctx).decode()
            raise TskvError(st, msg, self.lib.tskvgpu_last_error_page(self.ctx))

    def version(self):
        return self.lib.tskvgpu_version().decode()

    def comm_unique_id(self):
        """rank 0: the 128-byte NCCL unique id the other ranks need for comm_init."""
        buf = (C.c_uint8 * 128)()
        st = self.lib.tskvgpu_comm_unique_id(buf)
        if st != cabi.TSKV_OK:
            raise TskvError(st, "tskvgpu_comm_unique_id: NCCL unavailable")
        return bytes(buf)

    def comm_init(self, unique_id, rank, n_ranks):
        """ncclCommInitRank on this engine's device (collective: every rank calls it)."""
        buf = (C.c_uint8 * 128).from_buffer_copy(bytes(unique_id))
        self._check(self.lib.tskvgpu_comm_init(self.ctx, buf, int(rank), int(n_ranks)))

    def stream(self):
        return int(self.lib.tskvgpu_ctx_stream(self.ctx))

    def counters(self):
        c = cabi.Counters()
        self._check(self.lib.tskvgpu_get_counters(self.ctx, C.byref(c)))
        return {k: getattr(c, k) for k, _ in cabi.Counters._fields_ if k != "reserved"}

    def upload_pages(self, arena, descs, verify_crc=True, host_resident=False, verify_on_read=False):
        """arena: uint8 array (or (ptr, len)); descs: array of PAGE_DESC_DTYPE.
        host_resident=True keeps the page bytes in (page-locked) host memory: every scan then pulls the
        selected pages over PCIe itself; the caller must keep `arena` alive until PageSet.close().
        verify_on_read=True re-checks the CRC32 of every page a scan reads on the device, every scan."""
        if isinstance(arena, tuple):
            aptr, alen = arena
        else:
            arena = np.ascontiguousarray(arena, dtype=np.uint8)
            aptr, alen = arena.ctypes.data, arena.size
        descs = np.ascontiguousarray(descs, dtype=cabi.PAGE_DESC_DTYPE)
        h = C.c_void_p()
        flags = ((cabi.TSKV_UPLOAD_VERIFY_CRC if verify_crc else 0) | (cabi.TSKV_UPLOAD_HOST_RESIDENT if host_resident else 0) |
                 (cabi.TSKV_UPLOAD_VERIFY_ON_READ if verify_on_read else 0))
        st = self.lib.tskvgpu_upload_pages(self.ctx, aptr, alen, descs.ctypes.data, len(descs), flags, C.byref(h))
        self._check(st)
        ps = PageSet(self, h, len(descs))
        ps._keep = arena if host_resident else None
        return ps

    def decode_pages(self, pages, descs, first_page=0, n_pages=None):
        """Page::to_arrow_array for a page range: returns a list of (u64 values, bool validity)."""
        descs = np.ascontiguousarray(descs, dtype=cabi.PAGE_DESC_DTYPE)
        n_pages = len(descs) - first_page if n_pages is None else n_pages
        rows = descs["num_values"][first_page:first_page + n_pages].astype(np.uint64)
        bm = (rows + 63) // 64 * 8
        values = np.zeros(int(rows.sum()), dtype=np.uint64)
        bitmaps = np.zeros(int(bm.sum()), dtype=np.uint8)
        self._check(self.lib.tskvgpu_decode_pages(self.ctx, pages.handle, first_page, n_pages,
                                                  values.ctypes.data, bitmaps.ctypes.data))
        out, ro, bo = [], 0, 0
        for r, b in zip(rows, bm):
            r, b = int(r), int(b)
            valid = np.unpackbits(bitmaps[bo:bo + b], bitorder="little")[:r].astype(bool)
            out.append((values[ro:ro + r], valid))
            ro += r
            bo += b
        return out

    @staticmethod
    def _group_map(group_ids, n_groups):
        """GROUP BY tags arguments: (pointer or None, n_groups, array kept alive), or None for an ungrouped call.
        n_groups defaults to max(group_ids) + 1."""
        if group_ids is None and n_groups is None:
            return None
        ids = None if group_ids is None else np.ascontiguousarray(group_ids, dtype=np.uint32)
        if n_groups is None:
            n_groups = int(ids.max()) + 1 if ids is not None and ids.size else 1
        return (None if ids is None else ids.ctypes.data), int(n_groups), ids

    @staticmethod
    def _no_m2_with_slide(query, slide):
        if slide is not None and any(c.agg_mask & TSKV_AGG_M2 for c in query.columns):
            raise ValueError("m2 / var* / stddev* and slide: sliding windows do not push the variance state down")
        if slide is not None and getattr(query, "pairs", None):
            raise ValueError("pairs (covar* / corr) and slide: sliding windows do not push the covariance state down")
        if any(getattr(c, "median", False) for c in query.columns):
            if slide is not None:
                raise ValueError("median and slide: sliding windows do not push medians down")
            if getattr(query, "multi_rank", False):
                raise ValueError("median and multi_rank: medians have no mergeable partial state")
        if slide is not None and any(getattr(c, "increase", False) for c in query.columns):
            raise ValueError("increase and slide: sliding windows do not push increases down")

    @staticmethod
    def _edges(edges, slide):
        """Explicit time-bucket edges as a contiguous int64 array (kept alive by the caller), or None."""
        if edges is None:
            return None
        if slide is not None:
            raise ValueError("edges and slide: sliding windows over explicit time-bucket edges are not supported")
        return np.ascontiguousarray(edges, dtype=np.int64)

    @staticmethod
    def _labels(labels, edges):
        """Output bucket of every edge bucket as a contiguous uint32 array (kept alive by the caller), or None."""
        if labels is None:
            return None
        if edges is None:
            raise ValueError("labels need edges: label b names the output bucket of edge bucket b")
        lab = np.ascontiguousarray(labels, dtype=np.uint32)
        if lab.size != len(edges) - 1:
            raise ValueError("labels: one label per edge bucket (len(edges) - 1 = %d), got %d" % (len(edges) - 1, lab.size))
        return lab

    def output_layout(self, pages, query, group_ids=None, n_groups=None, edges=None, labels=None):
        L = cabi.OutputLayout()
        q = query.to_c()
        g = self._group_map(group_ids, n_groups)
        e = self._edges(edges, None)
        lab = self._labels(labels, e)
        if lab is not None:
            st = self.lib.tskvgpu_query_output_layout_labels(pages.handle, C.byref(q), e.ctypes.data, lab.size,
                                                             lab.ctypes.data, g[0] if g else None, g[1] if g else 0,
                                                             C.byref(L))
        elif e is not None:
            st = self.lib.tskvgpu_query_output_layout_edges(pages.handle, C.byref(q), e.ctypes.data,
                                                            g[0] if g else None, g[1] if g else 0, C.byref(L))
        elif g is None:
            st = self.lib.tskvgpu_query_output_layout(pages.handle, C.byref(q), C.byref(L))
        else:
            st = self.lib.tskvgpu_query_output_layout_grouped(pages.handle, C.byref(q), g[0], g[1], C.byref(L))
        if st != cabi.TSKV_OK:
            raise TskvError(st, "invalid query")
        return L

    def scan_aggregate(self, pages, query, slide=None, group_ids=None, n_groups=None, edges=None, labels=None):
        """End-to-end call: query args H2D, fused scan, result D2H (BatchReader::process analogue).
        slide: sliding windows time_window(time, query.width, slide, query.origin); output bucket j is the window
        starting at query.first_bucket_start + j * slide (sliding_window_grid sizes that grid).
        group_ids: GROUP BY tags, group_ids[slot] = group of the slot-th selected series (n_groups groups, default
        max + 1; the result has one row of buckets per group).
        edges: explicit time buckets [edges[b], edges[b + 1]) (query.n_buckets + 1 increasing timestamps, query.width,
        origin and first_bucket_start 0; calendar_edges makes them for date_trunc). Not with slide.
        labels: with edges, labels[b] < query.n_buckets is the output bucket of edge bucket b (one per edge bucket;
        calendar_parts makes them for date_part). query.n_buckets is then the number of output buckets."""
        self._no_m2_with_slide(query, slide)
        e = self._edges(edges, slide)
        lab = self._labels(labels, e)
        L = self.output_layout(pages, query, group_ids, n_groups, e, lab)
        values = np.empty(int(L.n_out * L.n_cells), dtype=np.uint64)
        bitmaps = np.empty(int(L.validity_bytes), dtype=np.uint8)
        g = self._group_map(group_ids, n_groups)
        q = query.to_c()
        if lab is not None:
            st = self.lib.tskvgpu_scan_aggregate_labels(self.ctx, pages.handle, C.byref(q), e.ctypes.data, lab.size,
                                                        lab.ctypes.data, g[0] if g else None, g[1] if g else 0,
                                                        values.ctypes.data, bitmaps.ctypes.data)
        elif e is not None:
            st = self.lib.tskvgpu_scan_aggregate_edges(self.ctx, pages.handle, C.byref(q), e.ctypes.data,
                                                       g[0] if g else None, g[1] if g else 0,
                                                       values.ctypes.data, bitmaps.ctypes.data)
        elif g is not None:
            st = self.lib.tskvgpu_scan_aggregate_grouped(self.ctx, pages.handle, C.byref(q), g[0], g[1], int(slide or 0),
                                                         values.ctypes.data, bitmaps.ctypes.data)
        elif slide is None:
            st = self.lib.tskvgpu_scan_aggregate(self.ctx, pages.handle, C.byref(q), values.ctypes.data, bitmaps.ctypes.data)
        else:
            st = self.lib.tskvgpu_scan_aggregate_sliding(self.ctx, pages.handle, C.byref(q), int(slide),
                                                         values.ctypes.data, bitmaps.ctypes.data)
        self._check(st)
        return ScanResult(query, L, values, bitmaps)

    def prepare(self, pages, query, slide=None, group_ids=None, n_groups=None, edges=None, labels=None):
        """Device-resident scan (run / enqueue / partials / exchange / finalize); slide, group_ids, edges, labels: as in
        scan_aggregate."""
        self._no_m2_with_slide(query, slide)
        e = self._edges(edges, slide)
        lab = self._labels(labels, e)
        L = self.output_layout(pages, query, group_ids, n_groups, e, lab)
        g = self._group_map(group_ids, n_groups)
        q = query.to_c()
        h = C.c_void_p()
        if lab is not None:
            st = self.lib.tskvgpu_scan_prepare_labels(self.ctx, pages.handle, C.byref(q), e.ctypes.data, lab.size,
                                                      lab.ctypes.data, g[0] if g else None, g[1] if g else 0, C.byref(h))
        elif e is not None:
            st = self.lib.tskvgpu_scan_prepare_edges(self.ctx, pages.handle, C.byref(q), e.ctypes.data,
                                                     g[0] if g else None, g[1] if g else 0, C.byref(h))
        elif g is not None:
            st = self.lib.tskvgpu_scan_prepare_grouped(self.ctx, pages.handle, C.byref(q), g[0], g[1], int(slide or 0), C.byref(h))
        elif slide is None:
            st = self.lib.tskvgpu_scan_prepare(self.ctx, pages.handle, C.byref(q), C.byref(h))
        else:
            st = self.lib.tskvgpu_scan_prepare_sliding(self.ctx, pages.handle, C.byref(q), int(slide), C.byref(h))
        self._check(st)
        return PreparedScan(self, pages, query, h, L)
