"""Exact per-cell gauge_agg(time, x) (TSKV_QUERY_N_GAUGES) for arenas described by a `truth` dict (tests/helpers.py
random_arena's), with median_reference.selected_values' row selection (covariance_reference.paired_rows with one
operand: series, time ranges, buckets, predicates, tombstones, merged rows of overlapping chunk files).

A cell's selected points (t, slot, v) are sorted by (t, slot) (slot: the series' position in the selection, FIRST /
LAST's tie rule; the reference leaves the order of equal timestamps unspecified) and give n and the points at positions
0, 1, n - 2 and n - 1 (gauge_agg.rs GaugeDataBuilder::build). Values convert to f64 as Rust's `as f64` does (nearest,
ties to even: numpy's conversion).

`update_batch_reference` restates the reference's update_batch + build over a split of the points into batches: each
batch keeps its first two and last two points (in input order) and the kept points are sorted by time at the end."""
import copy
import json
import os
import re

import numpy as np

from cnosdb_b200 import cabi
from cnosdb_b200.engine import GAUGE_OUTS, gauge_stat
from tests.covariance_reference import paired_rows
from tests.helpers import sliding_window

ROW = -1


def f64_bits(v, pt):
    """The u64 bit pattern of the f64 a typed value converts to."""
    if pt == cabi.TSKV_PT_F64:
        return int(np.float64(v).view(np.uint64))
    x = np.int64(v) if pt == cabi.TSKV_PT_I64 else np.uint64(v)
    return int(np.float64(x).view(np.uint64))


def selected_points(truth, query, col, pt, **kw):
    """{cell: [(t, slot, f64 bit pattern)]} of operand (col, pt), sorted by (t, slot)."""
    sel = [int(s) for s in query.series_ids] if query.series_ids is not None else sorted(truth)
    slot_of = {sid: k for k, sid in enumerate(sel)}
    ids, flat = {}, []
    for sid, cgs in truth.items():
        out = []
        for ts, cols in cgs:
            if col in cols:
                v, ok = cols[col]
                rows = np.arange(len(flat), len(flat) + len(v), dtype=np.int64)
                flat.extend((int(t), slot_of.get(sid, -1), f64_bits(x, pt)) for t, x in zip(ts, v))
                cols = dict(cols)
                cols[ROW] = (rows, np.asarray(ok, dtype=bool))
            out.append((ts, cols))
        ids[sid] = out
    cells = paired_rows(ids, query, (col, pt, ROW, cabi.TSKV_PT_I64), **kw)
    return {cell: sorted((flat[int(r)] for r in rows), key=lambda p: (p[0], p[1])) for cell, (_, rows) in cells.items()}


def gauge_of(points):
    """The 9 outputs (u64 bit patterns) and their validity of sorted points."""
    n = len(points)
    if n == 0:
        return [0] * 9, [True] + [False] * 8
    out = [n]
    for p in (points[0], points[min(1, n - 1)], points[max(n - 2, 0)], points[-1]):
        out += [p[0] & 0xFFFFFFFFFFFFFFFF, p[2]]
    return out, [True] * 9


def cells_from_points(pts, n_cells):
    """(values u64 [9, n_cells], validity bool [9, n_cells]) from {cell: sorted points}."""
    v = np.zeros((9, n_cells), dtype=np.uint64)
    ok = np.zeros((9, n_cells), dtype=bool)
    ok[0] = True
    for cell, p in pts.items():
        o, k = gauge_of(p)
        v[:, cell] = np.array(o, dtype=np.uint64)
        ok[:, cell] = k
    return v, ok


def exact_gauge_cells(truth, query, col, pt, n_cells, **kw):
    return cells_from_points(selected_points(truth, query, col, pt, **kw), n_cells)


def sliding_points(truth, query, col, pt, slide, n_groups, **kw):
    """{window cell: sorted points} of a sliding scan by row expansion: every selected point goes to each of its
    ceil(window / slide) windows (the reference's Expand plan) that lies on the grid first_bucket_start + j * slide."""
    flat = copy.copy(query)
    flat.width, flat.origin, flat.first_bucket_start, flat.n_buckets, flat._keep = 0, 0, 0, 1, None
    k = -(-query.width // slide)
    out = {}
    for group, pts in selected_points(truth, flat, col, pt, **kw).items():
        for p in pts:
            t = np.array([p[0]], dtype=np.int64)
            ws0, we0 = sliding_window(t, query.width, slide, query.origin, 0)
            if query.width % slide and not (ws0[0] <= t[0] < we0[0]):
                continue
            for i in range(k):
                ws, _ = sliding_window(t, query.width, slide, query.origin, i)
                d = int(ws[0]) - query.first_bucket_start
                if d < 0 or d % slide or d // slide >= query.n_buckets:
                    raise AssertionError("a window off the grid")
                out.setdefault(group * query.n_buckets + d // slide, []).append(p)
    return {c: sorted(v, key=lambda p: (p[0], p[1])) for c, v in out.items()}


def pane_points(truth, query, col, pt, slide, **kw):
    """{window cell: sorted points} by panes one slide wide folded k at a time (the scan's construction)."""
    k = -(-query.width // slide)
    panes = copy.copy(query)
    panes.width, panes.n_buckets, panes._keep = slide, query.n_buckets - k + 1, None
    panes.first_bucket_start = query.first_bucket_start + (k - 1) * slide
    out = {}
    for cell, pts in selected_points(truth, panes, col, pt, **kw).items():
        g, p = divmod(cell, panes.n_buckets)
        for j in range(p, min(p + k, query.n_buckets)):
            out.setdefault(g * query.n_buckets + j, []).extend(pts)
    return {c: sorted(v, key=lambda p: (p[0], p[1])) for c, v in out.items()}


def update_batch_reference(points, cuts):
    """gauge_agg.rs update_batch over batches points[cuts[i]:cuts[i + 1]] in input order: each batch is sorted by time
    (sort_to_indices) and keeps its points at positions 0, 1, len - 2 and len - 1; then GaugeDataBuilder::build sorts the
    kept points by time (a stable sort here; the reference's sort_unstable_by leaves ties in any order) -> (n, first,
    second, penultimate, last)."""
    kept, n = [], 0
    for a, b in zip(cuts[:-1], cuts[1:]):
        batch = sorted(points[a:b], key=lambda p: p[0])
        n += len(batch)
        if len(batch) <= 4:
            kept.extend(batch)
        else:
            kept.extend(batch[:2] + batch[-2:])
    if not kept:
        return 0, None, None, None, None
    kept.sort(key=lambda p: p[0])
    m = len(kept)
    return n, kept[0], kept[min(1, m - 1)], kept[max(m - 2, 0)], kept[-1]


def check_gauge(res, j0, exact, what=""):
    """Outputs j0 .. j0 + 8 of a ScanResult (one gauge) against exact_gauge_cells: validity equal, values bit for bit."""
    v_e, ok_e = exact
    for f in range(9):
        v, ok = res.values[j0 + f], res.validity[j0 + f]
        np.testing.assert_array_equal(ok, ok_e[f], err_msg="%s gauge %s validity" % (what, GAUGE_OUTS[f]))
        bad = np.nonzero(ok_e[f] & (v != v_e[f]))[0]
        assert bad.size == 0, (what, GAUGE_OUTS[f], [(int(i), hex(int(v[i])), hex(int(v_e[f][i]))) for i in bad[:5]])


def gauge_query_outputs(query):
    """The first output index of each gauge of `query` (they come last, 9 each, in column order)."""
    names = query.output_names()
    return [j for j, nm in enumerate(names) if nm[1] == "gauge_n"]


# ---- the reference's slt answers (tests/golden/gauge_slt.json, written by tests/golden/make_gauge_golden.py) ----------
GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "gauge_slt.json")
PT_OF = {"BIGINT": cabi.TSKV_PT_I64, "BIGINT UNSIGNED": cabi.TSKV_PT_U64, "DOUBLE": cabi.TSKV_PT_F64}
DAY = 86_400_000_000_000
_TOKEN = re.compile(r"\{.*?num_elements: \d+\}|-?\d+ years -?\d+ mons -?\d+ days -?\d+ hours -?\d+ mins -?[\d.]+ secs|\S+")
_ITEM = re.compile(r"(?:(\w+)\()?gauge_agg\(time, (\w+)(?: order by time)?\)\)?|\w+\([^)]*\)(?: - \w+\([^)]*\))?", re.I)


def load_golden():
    with open(GOLDEN) as f:
        return json.load(f)


def parse_ts(s):
    """ns of a printed or inserted timestamp ('1999-12-31T00:00:00.005', '1999-12-31 00:00:00.000', '100')."""
    s = s.strip().strip('"')
    if re.fullmatch(r"-?\d+", s):
        return int(s)
    return int(np.datetime64(s.replace(" ", "T"), "ns").astype(np.int64))


def parse_interval(s):
    """ns of a printed interval '0 years 0 mons 0 days 1 hours 0 mins 0.035000000 secs' (no years / months here)."""
    y, mo, d, h, mi, sec = re.fullmatch(r"(-?\d+) years (-?\d+) mons (-?\d+) days (-?\d+) hours (-?\d+) mins (-?[\d.]+) secs", s).groups()
    assert int(y) == 0 and int(mo) == 0, s
    whole, _, frac = sec.partition(".")
    return ((int(d) * 24 + int(h)) * 60 + int(mi)) * 60_000_000_000 + int(whole) * 1_000_000_000 + int((frac + "000000000")[:9])


def parse_struct(s):
    """(n, [(ts, val)] of first, second, penultimate, last) of a printed GaugeData."""
    pts = re.findall(r"(first|second|penultimate|last): \{ts: ([^,]+), val: ([^}]+)\}", s)
    return int(re.search(r"num_elements: (\d+)", s).group(1)), [(parse_ts(t), float(v)) for _, t, v in pts]


class GaugeGolden:
    """One answered query: its table's rows (t, series tags, {field: value or None}), the fields' types, the select items
    ((accessor or "gauge_agg", field) for a gauge item, None for another item), the grouping (None, "t0" or "day") and
    the expected tokens of every output row."""

    def __init__(self, g, a):
        self.src, self.sql = a["src"], a["sql"]
        tbl = g["tables"][a["table"]]
        cols, types = tbl["columns"], {k.lower(): v for k, v in tbl["types"].items()}
        tags = [c for c in cols if c != "time" and c not in types]
        rows = tbl["rows"][: a.get("n_rows") or len(tbl["rows"])]
        self.types = {c: PT_OF[t] for c, t in types.items() if t in PT_OF}
        self.rows = []
        for r in rows:
            d = dict(zip(cols, r))
            vals = {c: (None if d[c].lower() == "null" else (float(d[c]) if self.types[c] == cabi.TSKV_PT_F64 else int(d[c])))
                    for c in self.types if c in d}
            self.rows.append((parse_ts(d["time"]), tuple(d.get(t, "") for t in tags), vals))
        self.tags = tags
        sel = re.match(r"select (.*) from ", self.sql, flags=re.I).group(1)
        self.items = []
        for m in _ITEM.finditer(sel):
            self.items.append((m.group(1) or "gauge_agg", m.group(2).lower()) if m.group(2) else None)
        low = self.sql.lower()
        self.group = "t0" if "group by t0" in low else "day" if "date_trunc('day'" in low else None
        self.expected = [_TOKEN.findall(line) for line in a["expected"]]
        assert all(len(e) == len(self.items) for e in self.expected), (self.src, self.expected, self.items)

    def series(self):
        return sorted({tg for _, tg, _ in self.rows})

    def group_of(self, t, tg):
        if self.group == "t0":
            return tg[self.tags.index("t0")]
        return t // DAY if self.group == "day" else 0

    def groups(self):
        return sorted({self.group_of(t, tg) for t, tg, _ in self.rows})

    def reference_outputs(self, field):
        """[(n, first_t, first_v, second_t, ..., last_v)] per group: the exact reference on the golden table."""
        slot = {tg: k for k, tg in enumerate(self.series())}
        pt = self.types[field]
        out = []
        for grp in self.groups():
            pts = sorted((t, slot[tg], f64_bits(v[field], pt)) for t, tg, v in self.rows
                         if self.group_of(t, tg) == grp and v.get(field) is not None)
            out.append(decode_outputs(gauge_of(pts)[0]))
        return out

    def check(self, outputs):
        """outputs(field) -> [9-tuple per group] (decode_outputs'); every gauge item of every row against the answer."""
        for gi, row in enumerate(self.expected):
            for item, tok in zip(self.items, row):
                if item is None:
                    continue
                acc, field = item
                o = outputs(field)[gi]
                what = "%s %s row %d" % (self.src, acc, gi)
                if acc == "gauge_agg":
                    n, pts = parse_struct(tok)
                    assert o[0] == n, what
                    got = [(o[1], o[2]), (o[3], o[4]), (o[5], o[6]), (o[7], o[8])]
                    assert got == pts, (what, got, pts)
                    continue
                v, ok = gauge_stat(acc, *(np.array([x]) for x in o))
                assert bool(ok[0]), what
                if acc == "time_delta":
                    assert int(v[0]) == parse_interval(tok), (what, v[0], tok)
                elif acc in ("first_time", "last_time"):
                    assert int(v[0]) == parse_ts(tok), (what, v[0], tok)
                else:
                    assert np.isclose(float(v[0]), float(tok), rtol=1e-12, atol=0), (what, v[0], tok)


def decode_outputs(o):
    """The 9 outputs as u64 bit patterns -> (n, then t as int and v as float per point)."""
    out = [int(o[0])]
    for k in range(1, 9):
        out.append(int(np.uint64(o[k]).view(np.int64)) if k % 2 else float(np.uint64(o[k]).view(np.float64)))
    return tuple(out)


def golden_cases():
    g = load_golden()
    return [GaugeGolden(g, a) for a in g["answers"]]


def golden_refused():
    """The operand types gauge_agg refuses at planning: {'Boolean', 'Utf8', 'Timestamp'}."""
    return sorted({r["type"] for r in load_golden()["refused"]})
