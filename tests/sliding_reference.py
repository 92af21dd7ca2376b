"""Exact references for sliding windows, time_window(time, window, slide, start_time), from the generated arrays (no page
is decoded):
  expand_aggregate  a literal restatement of the reference's Expand plan (build_sliding_window_plan,
                    transform_time_window.rs:328-393): k = ceil(window / slide) copies of every selected row, copy i in the
                    window starting at last_start(t) - i * slide, the window-0 filter when window % slide != 0, and every
                    kept copy's window on the grid first_bucket_start + j * slide (j < n_buckets);
  pane_aggregate    the engine's method: each selected row once, in its pane (tumbling buckets of width `slide`, start
                    time % window), on the pane grid, then counted in the k windows that fold that pane.
Both aggregate with tests.helpers.exact_aggregate, so COUNT / SUM / MIN / MAX / MEAN follow its exact rules."""
import numpy as np

from cnosdb_b200 import cabi
from cnosdb_b200.engine import QueryOption
from tests.helpers import I64_MAX, I64_MIN, ReferenceError, _cmp, exact_aggregate, sliding_window, wrap64


def n_windows_per_row(window, slide):
    return -(-window // slide)


def _cmod(a, b):
    r = abs(a) % abs(b)
    return -r if a < 0 else r


def _selected(ts, cols, query):
    """Rows the time ranges and AND-ed predicates select (NULL or an absent predicate column: not selected)."""
    sel = np.ones(ts.size, dtype=bool)
    for pc, ppt, op, c in query.predicates:
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
    return sel


def _grid_index(starts, first, n, slide):
    """(index, on the grid) of window starts: first + j * slide, 0 <= j < n (wrapping difference, like the scan)."""
    with np.errstate(over="ignore"):
        diff = starts - np.int64(wrap64(first))
    idx = np.where(diff >= 0, diff // np.int64(slide), -1)
    return idx, (diff >= 0) & (np.fmod(diff, np.int64(slide)) == 0) & (idx < n)


def _aggregate_copies(truth, query, copies_of):
    """exact_aggregate over the window copies: copies_of(ts, selected) -> [(row indices, window index)] per column group."""
    expanded = {}
    for sid, cgs in truth.items():
        out = []
        for ts, cols in cgs:
            ts = np.asarray(ts, dtype=np.int64)
            rows = np.nonzero(_selected(ts, cols, query))[0]
            for r, j in copies_of(ts[rows]):
                rr = rows[r]
                out.append((np.asarray(j, dtype=np.int64),
                            {c: (np.asarray(v)[rr], np.asarray(ok, dtype=bool)[rr]) for c, (v, ok) in cols.items()}))
        expanded[sid] = out
    windows = QueryOption(query.columns, series_ids=query.series_ids, width=1, origin=0, first_bucket_start=0,
                          n_buckets=query.n_buckets, group_by_series=query.group_by_series)
    return exact_aggregate(expanded, windows)


def expand_aggregate(truth, query, slide):
    """The Expand plan, row copy by row copy. Raises ReferenceError(TSKV_ERR_BUCKET_RANGE) when a kept copy's window is
    not on the grid."""
    window, origin = query.width, query.origin
    k = n_windows_per_row(window, slide)

    def copies(t):
        ws0, we0 = sliding_window(t, window, slide, origin, 0)
        keep = np.ones(t.size, dtype=bool) if window % slide == 0 else (t >= ws0) & (t < we0)
        out = []
        for i in range(k):
            ws, _ = sliding_window(t, window, slide, origin, i)
            j, ok = _grid_index(ws, query.first_bucket_start, query.n_buckets, slide)
            if (keep & ~ok).any():
                raise ReferenceError(cabi.TSKV_ERR_BUCKET_RANGE)
            out.append((np.nonzero(keep)[0], j[keep]))
        return out
    return _aggregate_copies(truth, query, copies)


def pane_aggregate(truth, query, slide):
    """Tumbling panes of width `slide` on the grid first_bucket_start + (k - 1) * slide + p * slide, p < n_buckets - k + 1,
    each folded into windows p .. p + k - 1. Raises ReferenceError(TSKV_ERR_BUCKET_RANGE) for a row without a pane."""
    window, origin = query.width, query.origin
    k = n_windows_per_row(window, slide)

    def copies(t):
        start, _ = sliding_window(t, window, slide, origin, 0)  # the pane: t - ((t - origin % window) + slide) % slide
        p, ok = _grid_index(start, query.first_bucket_start + (k - 1) * slide, query.n_buckets - k + 1, slide)
        if not ok.all():
            raise ReferenceError(cabi.TSKV_ERR_BUCKET_RANGE)
        return [(np.arange(t.size), p + i) for i in range(k)]
    return _aggregate_copies(truth, query, copies)


def sliding_status(truth, query, slide):
    """The status tskvgpu_scan_prepare_sliding refuses `query` with (None: accepted), in the library's order."""
    w, nb = query.width, query.n_buckets
    if slide <= 0 or w <= 0:
        return cabi.TSKV_ERR_INVALID_ARG
    if slide == w:
        return None
    if any(c.agg_mask & (cabi.TSKV_AGG_FIRST | cabi.TSKV_AGG_LAST) for c in query.columns):
        return cabi.TSKV_ERR_UNSUPPORTED
    if slide > w or w >= 2**61:
        return cabi.TSKV_ERR_UNSUPPORTED
    k = n_windows_per_row(w, slide)
    if k > 100 or nb < k or nb * slide > 2**63:
        return cabi.TSKV_ERR_INVALID_ARG
    if w % slide:
        lo = min(int(ts.min()) for cgs in truth.values() for ts, _ in cgs if len(ts))
        hi = max(int(ts.max()) for cgs in truth.values() for ts, _ in cgs if len(ts))
        if query.time_ranges:
            lo = max(lo, min(a for a, _ in query.time_ranges))
            hi = min(hi, max(b for _, b in query.time_ranges))
        om = _cmod(query.origin, w)
        if lo <= hi and (lo - om + slide < 0 or hi - om + slide > I64_MAX or hi + w > I64_MAX):
            return cabi.TSKV_ERR_UNSUPPORTED
    return None


def sliding_fit_grid(truth, window, slide, origin, ranges, max_windows=1 << 22):
    """(first_bucket_start, n_buckets) of the smallest window grid holding every window of every row the ranges select,
    leaving out rows whose window arithmetic wraps (those must get TSKV_ERR_BUCKET_RANGE); (0, k) when no row is
    selected, None when the grid would exceed max_windows."""
    k = n_windows_per_row(window, slide)
    om = _cmod(origin, window)
    lo_starts, hi_starts = [], []
    for cgs in truth.values():
        for ts, _ in cgs:
            t = np.asarray(ts, dtype=np.int64)
            if ranges:
                sel = np.zeros(t.size, dtype=bool)
                for a, b in ranges:
                    sel |= (t >= a) & (t <= b)
                t = t[sel]
            if t.size == 0:
                continue
            # every step of last_start(t) - (k - 1) * slide without wrapping
            ok = (t <= I64_MAX + om) if om < 0 else (t >= I64_MIN + om)
            with np.errstate(over="ignore"):
                d = t - np.int64(om)
                ok &= d <= np.int64(I64_MAX - slide)
                ls, _ = sliding_window(t, window, slide, origin, 0)
                rem = t - ls
            ok &= np.where(rem > 0, t >= I64_MIN + np.maximum(rem, 0), t <= I64_MAX + np.minimum(rem, 0))
            ok &= ls >= np.int64(I64_MIN + (k - 1) * slide)
            if ok.any():
                lo_starts.append(int(ls[ok].min()) - (k - 1) * slide)
                hi_starts.append(int(ls[ok].max()))
    if not lo_starts:
        return 0, k
    first, last = min(lo_starts), max(hi_starts)
    nb = (last - first) // slide + 1
    return (first, nb) if nb <= max_windows else None
