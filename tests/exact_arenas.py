"""Arenas aimed at the row semantics the exact reference of tests/helpers.py restates: FIRST / LAST runs, tombstone range
edges and the overlap merge of chunk files. Each builder returns what the exact reference and the oracle both take, so
tests/test_exact_reference.py checks the reference against the oracle on every arena here (no GPU), and
tests/test_gpu_first_last_tombstones.py / tests/test_gpu_merge_exact.py check the scan against the reference."""
import numpy as np

from cnosdb_b200 import cabi, datagen
from cnosdb_b200.engine import PushedAggregate, QueryOption, sliding_window_grid
from tests.helpers import (ALL_AGGS, I64_MAX, I64_MIN, _merged_rows, _typed, bucket_spec, exact_aggregate,
                           overlap_groups, sliding_window)

SEL_AGGS = ("count", "min", "max", "first", "last")  # (booleans: no SUM / MEAN)
PLAIN_AGGS = ("count", "sum", "min", "max", "mean")


def add_column_group(b, sid, ts, fields, raw_time=False):
    """ArenaBuilder.add_column_group, or with raw_time the same column group behind a raw (Encoding::Null) time page:
    the scan's generic-time kernels."""
    if not raw_time:
        b.add_column_group(sid, ts, fields)
        return
    n = len(ts)
    b.add_page(datagen.build_page(datagen.encode_raw(np.asarray(ts, dtype=np.int64)), n), sid, 0, cabi.TSKV_PT_TIME, n)
    for f in fields:
        col, pt, vals, valid = f[:4]
        enc = f[4] if len(f) > 4 and f[4] is not None else (
            datagen.encode_floats if pt == cabi.TSKV_PT_F64 else datagen.encode_bools if pt == cabi.TSKV_PT_BOOL
            else datagen.encode_integers)
        vals = np.asarray(vals)
        kept = vals if valid is None else vals[np.asarray(valid, dtype=bool)]
        if pt == cabi.TSKV_PT_U64 and enc is datagen.encode_integers:
            kept = np.asarray(kept, dtype=np.uint64).view(np.int64)
        b.add_page(datagen.build_page(enc(kept), n, valid), sid, col, pt, n)


def _values(rng, pt, n, wide):
    if pt == cabi.TSKV_PT_F64:
        return np.cumsum(rng.integers(-3, 4, n)).astype(np.float64) + rng.random(n)
    if pt == cabi.TSKV_PT_U64:
        return (rng.integers(0, 2**62, n, dtype=np.uint64) + np.uint64(2**63)) if wide else \
            rng.integers(0, 1000, n).astype(np.uint64)
    if pt == cabi.TSKV_PT_BOOL:
        return rng.random(n) < 0.5
    return rng.integers(-2**62, 2**62, n) if wide else np.cumsum(rng.integers(-3, 4, n)).astype(np.int64)


# ---- FIRST / LAST ------------------------------------------------------------------------------------------------------
# 20 series on a grid of STEP-spaced rows, buckets of 10 rows starting at T0: column groups of 37, 130 and 64 rows, so
# runs of one series start and end inside buckets. Columns: 1 i64 (narrow / wide simple8b), 2 f64 (Gorilla), 3 u64
# (narrow / wide), 4 i64 raw (-1 on bucket-first rows of every third series: the predicate 4 >= 0 drops them), 5 bool.
# Nulls by sid % 4: 1 at every bucket's first row, 2 at its last row, 3 at random; 0 none. Times by kind: "rle" the grid
# (every series shares it: equal times across slots), "s8b" jittered (even series share their jitter), "raw" the grid
# behind raw time pages.

FL_T0, FL_STEP, FL_W = 10**12, 1000, 10_000
FL_SERIES = 20
FL_FIELDS = ((1, cabi.TSKV_PT_I64), (2, cabi.TSKV_PT_F64), (3, cabi.TSKV_PT_U64), (4, cabi.TSKV_PT_I64),
             (5, cabi.TSKV_PT_BOOL))
FL_KINDS = ("rle", "s8b", "raw")


def first_last_arena(kind, seed=1):
    rng = np.random.default_rng(seed + FL_KINDS.index(kind))
    shared_jit = rng.integers(0, FL_STEP, 400)
    b = datagen.ArenaBuilder()
    truth = {}
    for sid in range(FL_SERIES):
        k0 = sid % 3
        for n in ((37, 130, 64)[: 1 + sid % 3]):
            k = k0 + np.arange(n)
            k0 += n + 1 + sid % 2
            ts = FL_T0 + k * FL_STEP
            if kind == "s8b":
                jit = shared_jit[k % 400] if sid % 2 == 0 else rng.integers(0, FL_STEP, n)
                ts = ts + np.where(k % 10 == 0, 0, jit)
            fl, cols = [], {}
            for col, pt in FL_FIELDS:
                vals = _values(rng, pt, n, wide=(sid // 2) % 2 == 1)
                if col == 4:
                    vals = np.where((k % 10 == 0) & (sid % 3 == 0), -1, np.abs(vals))
                valid = np.ones(n, dtype=bool)
                if sid % 4 == 1:
                    valid = k % 10 != 0
                elif sid % 4 == 2:
                    valid = k % 10 != 9
                elif sid % 4 == 3:
                    valid = rng.random(n) >= 0.3
                if col == 4:
                    valid = np.ones(n, dtype=bool)
                enc = datagen.encode_raw if col == 4 else None
                fl.append((col, pt, vals, None if valid.all() else valid, enc))
                cols[col] = (vals, valid)
            add_column_group(b, sid, ts, fl, raw_time=kind == "raw")
            truth.setdefault(sid, []).append((ts, cols))
    arena, descs = b.finish()
    return arena, descs, truth


def sel_columns(fields, aggs=ALL_AGGS):
    return [PushedAggregate(c, pt, SEL_AGGS if pt == cabi.TSKV_PT_BOOL else aggs) for c, pt in fields]


def first_last_queries(truth):
    """[(name, query, extra)]: extra = {} or {"group_ids", "n_groups"} (GROUP BY tags)."""
    t_hi = max(int(ts.max()) for cgs in truth.values() for ts, _ in cgs)
    fbs, nb = bucket_spec(FL_T0, t_hi, FL_W)
    grid = dict(width=FL_W, first_bucket_start=fbs, n_buckets=nb)
    cols = sel_columns(FL_FIELDS)
    ends = np.array([0, 1, 5, 7, 11, FL_SERIES - 1], dtype=np.uint32)  # the lowest and highest selected slot
    ranges = [(FL_T0 + 15 * FL_STEP + 1, FL_T0 + 95 * FL_STEP), (FL_T0 + 120 * FL_STEP, FL_T0 + 121 * FL_STEP - 1)]
    ids = np.arange(FL_SERIES, dtype=np.uint32)
    return [
        ("bucket", QueryOption(cols, **grid), {}),
        ("ranges", QueryOption(cols, time_ranges=ranges, **grid), {}),
        ("predicate", QueryOption(cols, predicates=[(4, cabi.TSKV_PT_I64, ">=", 0)], **grid), {}),
        ("ends", QueryOption(cols, series_ids=ends, **grid), {}),
        ("by_series", QueryOption(cols, group_by_series=True, **grid), {}),
        ("by_series_pred", QueryOption(cols, group_by_series=True, predicates=[(4, cabi.TSKV_PT_I64, ">=", 0)],
                                       time_ranges=ranges, **grid), {}),
        ("unbucketed", QueryOption(cols), {}),
        ("unbucketed_ranges", QueryOption(cols, time_ranges=ranges), {}),
        ("tags", QueryOption(cols, **grid), {"group_ids": (ids * 7 % 3).astype(np.uint32), "n_groups": 3}),
    ]


# The 62-bit key budget: three series (slot_bits 2) with rows at both ends of `rel` (a bucket's first and last ns), at
# widths where bits(2 * width) + 2 is 61, 62 and 63; unbucketed, page-set spans of 2^60 - 1 and 2^60.

BUDGET_WIDTHS = ((2**58 - 1, 61), (2**59 - 1, 62), (2**59, 63))


def key_budget_arena(width, unbucketed_span=None):
    """Rows at 0, width - 1, width, 2 width - 1 (bucket ends) for slots 0-2; unbucketed_span: rows at 0 and the span."""
    b = datagen.ArenaBuilder()
    truth = {}
    if unbucketed_span is None:
        ts = np.array([0, 1, width - 1, width, width + 5, 2 * width - 1], dtype=np.int64)
    else:
        ts = np.array([0, 3, unbucketed_span // 2, unbucketed_span - 1, unbucketed_span], dtype=np.int64)
    for sid in range(3):
        n = ts.size
        vals = np.arange(n, dtype=np.int64) * 10 + sid
        valid = np.ones(n, dtype=bool)
        valid[(sid + np.arange(n)) % 3 == 0] = False  # slots take turns holding the value at each time
        b.add_column_group(sid, ts, [(1, cabi.TSKV_PT_I64, vals, valid)])
        truth[sid] = [(ts, {1: (vals, valid)})]
    arena, descs = b.finish()
    return arena, descs, truth


def key_budget_queries(width, unbucketed=False):
    cols = [PushedAggregate(1, cabi.TSKV_PT_I64, ("count", "first", "last"))]
    if unbucketed:
        return [("unbucketed", QueryOption(cols), {})]
    return [("bucket", QueryOption(cols, width=width, first_bucket_start=0, n_buckets=2), {})]


# ---- tombstones --------------------------------------------------------------------------------------------------------
# Series 0-9 on a grid of `step` (RLE time pages, simple8b ones with jitter below the step, or raw ones: the generic-time
# kernels), page lengths 300, 1000, 129 and 1 (restart points every 128 rows: the cuts of pages in parts), columns 1 i64
# narrow, 2 i64 wide, 3 i64 mixed (narrow with a wide value every ~50 rows), 4 f64. Series 10 starts at INT64_MIN,
# series 11 ends at INT64_MAX.

TB_T0 = 10**12
TB_FIELDS = ((1, cabi.TSKV_PT_I64), (2, cabi.TSKV_PT_I64), (3, cabi.TSKV_PT_I64), (4, cabi.TSKV_PT_F64))
TB_CASES = ((1, "rle"), (3, "rle"), (3, "s8b"), (3, "raw"))
TB_LENGTHS = (300, 1000, 129, 1)
TB_LIMIT_SERIES = (10, 11)


def tomb_width(step):
    return 37 * step


def tombstone_arena(step, kind, seed=5):
    rng = np.random.default_rng(seed + step + len(kind))
    b = datagen.ArenaBuilder()
    truth = {}
    for sid in range(12):
        n = TB_LENGTHS[sid % 4] if sid < 10 else 200
        k = np.arange(n, dtype=np.int64)
        if sid == 10:
            ts = I64_MIN + k * step
        elif sid == 11:
            ts = I64_MAX - (n - 1 - k) * step
        else:
            ts = TB_T0 + (sid % 3) * step + k * step
            if kind == "s8b" and n > 2:
                ts = ts + np.where((k == 0) | (k == n - 1), 0, rng.integers(0, step, n))
        fl, cols = [], {}
        for col, pt in TB_FIELDS:
            if col == 3:
                vals = np.cumsum(rng.integers(-3, 4, n)).astype(np.int64)
                vals[rng.random(n) < 0.02] = 2**61 + 5
            else:
                vals = _values(rng, pt, n, wide=col == 2)
            valid = rng.random(n) >= 0.1 if sid % 3 == 1 else np.ones(n, dtype=bool)
            fl.append((col, pt, vals, None if valid.all() else valid))
            cols[col] = (vals, valid)
        add_column_group(b, sid, ts, fl, raw_time=kind == "raw")
        truth[sid] = [(ts, cols)]
    arena, descs = b.finish()
    return arena, descs, truth


def tombstone_list(truth, step, seed=9):
    """Ranges whose edges lie on a row, one before it or one after it, at bucket starts / ends, the restart-point cuts
    (rows 127-129, 255-257), page ends and the i64 limits; 40 ranges on two keys, nested and overlapping ranges, keys of
    series and columns that do not exist, and empty ranges."""
    rng = np.random.default_rng(seed + step)
    w = tomb_width(step)
    out = []
    for sid in range(10):
        ts = truth[sid][0][0]
        n = ts.size
        rows = sorted({r for r in (0, 1, 127, 128, 129, 255, 256, 257, n - 2, n - 1) if 0 <= r < n})
        starts, _ = sliding_window(ts, w, w, 0)
        rows += list(np.flatnonzero(ts == starts)[:4]) + list(np.flatnonzero(ts == starts + w - step)[:4])
        for _ in range(8):
            a, bb = sorted(rng.choice(rows, 2))
            da, db = (int(x) for x in rng.integers(-1, 2, 2))
            lo, hi = int(ts[a]) + da, int(ts[bb]) + db
            r = rng.random()
            col = None if r < 0.35 else int(rng.integers(1, 5))
            out.append((None if r < 0.05 else sid, None if r < 0.05 else col, lo, hi))
    t = truth[0][0][0]
    out += [(0, 1, int(t[7 * i]), int(t[7 * i + 2])) for i in range(40)]            # > 32 ranges on one key
    t = truth[1][0][0]
    out += [(1, None, int(t[20 * i + 3]) - 1, int(t[20 * i + 3]) + 1) for i in range(40)]
    t = truth[5][0][0]
    out += [(5, 2, int(t[10]), int(t[50])), (5, 2, int(t[20]), int(t[30])),         # nested
            (5, None, int(t[60]), int(t[80])), (5, None, int(t[70]), int(t[90])),   # overlapping
            (999, None, I64_MIN, I64_MAX), (3, 77, I64_MIN, I64_MAX),               # no such series / column
            (4, 1, int(t[9]), int(t[3])), (None, None, int(t[5]), int(t[4]))]       # empty
    lo_t, hi_t = truth[10][0][0], truth[11][0][0]
    out += [(10, None, I64_MIN, I64_MIN), (10, 1, I64_MIN, int(lo_t[5])), (11, None, I64_MAX, I64_MAX),
            (11, 4, int(hi_t[-4]), I64_MAX), (None, None, I64_MIN, I64_MIN + step)]
    return cabi.tombstones(out)


def tombstone_queries(truth, step):
    w = tomb_width(step)
    normal = np.arange(10, dtype=np.uint32)
    t_hi = max(int(truth[s][0][0].max()) for s in range(10))
    fbs, nb = bucket_spec(TB_T0, t_hi, w)
    grid = dict(width=w, first_bucket_start=fbs, n_buckets=nb)
    cols = sel_columns(TB_FIELDS)
    plain = [PushedAggregate(c, pt, PLAIN_AGGS) for c, pt in TB_FIELDS]
    return [
        ("bucket", QueryOption(cols, series_ids=normal, **grid), {}),
        ("by_series", QueryOption(cols, series_ids=normal, group_by_series=True, **grid), {}),
        ("ranges", QueryOption(cols, series_ids=normal, time_ranges=[(TB_T0 + 40 * step, TB_T0 + 700 * step)], **grid), {}),
        ("unbucketed_all", QueryOption(plain), {}),
        ("by_series_all", QueryOption(cols, group_by_series=True), {}),
        ("tags", QueryOption(cols, series_ids=normal, **grid), {"group_ids": (normal % 4).astype(np.uint32), "n_groups": 4}),
    ]


# ---- the overlap merge -------------------------------------------------------------------------------------------------
# Every series holds chunks of several files (file id per column group), on a STEP grid with bucket width MG_W and
# origin 3. Scenario by sid % 8:
#   0  2-8 files over one common span, duplicate times inside chunks (a run of 320 equal times in series 0 and 8)
#   1  a chain: A overlaps B, B overlaps C, A does not overlap C
#   2  two chunks touching at one timestamp (one group) ...
#   3  ... and two separated by a gap of 1 ns (two groups): FIRST of the bucket differs between 2 and 3
#   4  the newest chunk lacks column 2 and holds NULLs in column 1: older values show through
#   5  merged rows exactly on bucket starts / ends (origin 3) whose merged column-1 value is NULL
#   6  the newest chunk is a raw "memcache" chunk
#   7  a single file (the plain path)
# Series 40 / 41 lie at the i64 limits (chunks at INT64_MIN / INT64_MAX), selected only by the unbucketed queries.

MG_T0, MG_STEP, MG_W, MG_ORIGIN = 10**9, 1000, 17_000, 3
MG_FIELDS = ((1, cabi.TSKV_PT_I64), (2, cabi.TSKV_PT_F64), (3, cabi.TSKV_PT_U64))
MG_SERIES = 40
MG_LIMITS = (40, 41)


def _chunk_fields(rng, n, drop=(), null1=False, raw=False):
    fl, cols = [], {}
    for col, pt in MG_FIELDS:
        if col in drop:
            continue
        valid = rng.random(n) >= 0.25
        if null1 and col == 1:
            valid = np.zeros(n, dtype=bool) if rng.random() < 0.5 else rng.random(n) < 0.1
        vals = _values(rng, pt, n, wide=rng.random() < 0.3)
        fl.append((col, pt, vals, valid, datagen.encode_raw if raw else None))
        cols[col] = (vals, valid)
    return fl, cols


def merge_arena(seed=3):
    """-> (arena, descs, truth, files): files[k] the file id of the k-th column group in truth's order."""
    rng = np.random.default_rng(seed)
    b = datagen.ArenaBuilder()
    truth, files = {}, []

    def add(sid, fid, ts, fl, cols):
        b.add_column_group(sid, np.asarray(ts, dtype=np.int64), fl)
        truth.setdefault(sid, []).append((np.asarray(ts, dtype=np.int64), cols))
        files.append(fid)

    g = lambda k: MG_T0 + np.asarray(k, dtype=np.int64) * MG_STEP  # noqa: E731
    for sid in range(MG_SERIES):
        sc = sid % 8
        if sc == 0:
            nf = 2 + (sid // 8) * 3 % 7  # 2, 5, 8, 4, 7 files
            for f in range(nf):
                n = int(rng.integers(100, 300))
                k = np.sort(rng.integers(0, 260, n))  # duplicates inside the chunk
                if f == 0 and sid in (0, 8):
                    k = np.sort(np.concatenate([k[:20], np.full(320, 130)]))
                fl, cols = _chunk_fields(rng, k.size)
                add(sid, 10 * (f + 1) + sid % 3, g(k), fl, cols)
        elif sc == 1:
            for f, (a, z) in enumerate(((0, 100), (90, 200), (190, 300))):
                k = np.arange(a, z + 1)
                fl, cols = _chunk_fields(rng, k.size)
                add(sid, (3, 1, 2)[f], g(k), fl, cols)
        elif sc in (2, 3):
            k1 = np.arange(0, 51)
            fl, cols = _chunk_fields(rng, k1.size)
            add(sid, 2, g(k1), fl, cols)
            t2 = g(np.arange(50, 120)) + (1 if sc == 3 else 0)  # starts at chunk 1's last row / 1 ns after it
            fl, cols = _chunk_fields(rng, t2.size, null1=True)
            cols[1][1][0] = False
            fl[0] = (1, cabi.TSKV_PT_I64, cols[1][0], cols[1][1], None)
            add(sid, 1, t2, fl, cols)
        elif sc == 4:
            for f in range(3):
                k = np.arange(10 * f, 150 + 10 * f)
                fl, cols = _chunk_fields(rng, k.size, drop=(2,) if f == 2 else (), null1=f == 2)
                add(sid, 5 + f, g(k), fl, cols)
        elif sc == 5:
            starts = MG_ORIGIN + (MG_T0 // MG_W + np.arange(1, 12)) * MG_W
            t = np.unique(np.concatenate([starts, starts - 1, starts + 1, g(np.arange(0, 140, 3))]))
            for f in range(2):
                fl, cols = _chunk_fields(rng, t.size)
                edge = np.isin(t, np.concatenate([starts, starts - 1]))
                cols[1][1][edge] = False  # NULL in both chunks: the merged value is NULL
                fl[0] = (1, cabi.TSKV_PT_I64, cols[1][0], cols[1][1], None)
                add(sid, f + 1, t, fl, cols)
        elif sc == 6:
            for f in range(3):
                k = np.arange(20 * f, 120 + 20 * f)
                fl, cols = _chunk_fields(rng, k.size, raw=f == 2)
                add(sid, 100 + f, g(k), fl, cols)
        else:
            for part in range(2):
                k = np.arange(150 * part, 150 * part + 120)
                fl, cols = _chunk_fields(rng, k.size)
                add(sid, 9, g(k), fl, cols)
    for sid, base in zip(MG_LIMITS, (I64_MIN, I64_MAX - 198)):
        for f in range(3):
            k = np.sort(rng.integers(0, 100, 80)) * 2 + (f if base == I64_MIN else 0)
            fl, cols = _chunk_fields(rng, k.size)
            add(sid, f + 1, base + k, fl, cols)
    arena, descs = b.finish()
    return arena, descs, truth, np.array(files, dtype=np.uint64)


def merge_tombstones(truth):
    """Row and column tombstones at merged rows. Range edges avoid times that repeat inside one column group: there the
    reference's binary search over a page's times (which the oracle keeps) may stop inside the run of equal times,
    while the scan drops every row of the range (DESIGN section 7)."""
    def edges(sid):
        ts = np.unique(np.concatenate([t for t, _ in truth[sid]]))
        return ts[[all(np.count_nonzero(t == x) <= 1 for t, _ in truth[sid]) for x in ts]]
    out = []
    for sid in range(0, MG_SERIES, 3):
        ts = edges(sid)
        a, z = int(ts[len(ts) // 4]), int(ts[len(ts) // 4 + 5])
        out += [(sid, None, a, a), (sid, 1, z, int(ts[len(ts) // 2])), (sid, 2, a - 1, z + 1)]
    hi = edges(MG_LIMITS[1])
    out += [(None, None, MG_T0 + 200 * MG_STEP - 1, MG_T0 + 203 * MG_STEP + 1), (41, 1, int(hi[-4]), int(hi[-1])),
            (41, None, int(hi[-1]), int(hi[-1])), (40, None, I64_MIN, int(edges(MG_LIMITS[0])[2]))]
    return cabi.tombstones(out)


def merge_queries(truth):
    fbs, nb = bucket_spec(MG_T0 - MG_W, MG_T0 + 320 * MG_STEP, MG_W, origin=MG_ORIGIN)
    grid = dict(width=MG_W, origin=MG_ORIGIN, first_bucket_start=fbs, n_buckets=nb)
    ids = np.arange(MG_SERIES, dtype=np.uint32)
    sub = ids[ids % 5 != 2]
    cols = sel_columns(MG_FIELDS)
    rng_ = [(MG_T0 + 20 * MG_STEP, MG_T0 + 133 * MG_STEP - 1), (MG_T0 + 180 * MG_STEP + 1, MG_T0 + 290 * MG_STEP)]
    preds = [(1, cabi.TSKV_PT_I64, ">", -2**40)]  # drops the wide negative values of some chunks, nothing else
    return [
        ("bucket", QueryOption(cols, series_ids=ids, **grid), {}),
        ("by_series", QueryOption(cols, series_ids=ids, group_by_series=True, **grid), {}),
        ("subset_ranges", QueryOption(cols, series_ids=sub, time_ranges=rng_, **grid), {}),
        ("predicate", QueryOption(cols, series_ids=ids, predicates=preds, **grid), {}),
        ("by_series_predicate", QueryOption(cols, series_ids=ids, group_by_series=True, predicates=preds, **grid), {}),
        ("unbucketed", QueryOption(cols, series_ids=ids, time_ranges=[(MG_T0, MG_T0 + 400 * MG_STEP)]), {}),
        ("unbucketed_limits", QueryOption(cols, group_by_series=True), {}),
        ("tags", QueryOption(cols, series_ids=ids, **grid), {"group_ids": (ids % 3).astype(np.uint32), "n_groups": 3}),
    ]


def merge_sliding_query():
    """Windows of 3 buckets sliding by one (no FIRST / LAST: sliding scans refuse them)."""
    fbs, nb = sliding_window_grid(MG_T0 - MG_W, MG_T0 + 320 * MG_STEP, 3 * MG_W, MG_W, MG_ORIGIN)
    cols = [PushedAggregate(c, pt, PLAIN_AGGS) for c, pt in MG_FIELDS]
    return QueryOption(cols, series_ids=np.arange(MG_SERIES, dtype=np.uint32), width=3 * MG_W, origin=MG_ORIGIN,
                       first_bucket_start=fbs, n_buckets=nb, time_ranges=[(MG_T0 - MG_W, MG_T0 + 320 * MG_STEP)]), \
        {"slide": MG_W}


def merge_truth(truth, files, query):
    """truth with every overlap group of two or more chunks replaced by its merged rows (one column group): what a
    reference without a merge (sliding windows) takes. No predicates or tombstones."""
    assert not query.predicates
    qcols = [c.column_id for c in query.columns]
    out, k = {}, 0
    for sid, cgs in truth.items():
        fl = files[k:k + len(cgs)]
        k += len(cgs)
        out[sid] = []
        for streams in overlap_groups(cgs, fl):
            if len(streams) < 2:
                out[sid] += [cgs[j] for j in streams[0]]
                continue
            ts, cols = _merged_rows(cgs, streams, query, qcols, [])
            out[sid].append((ts, {c: (v.view(_typed(next(q.phys_type for q in query.columns if q.column_id == c), []).dtype), ok)
                                  for c, (v, ok) in cols.items()}))
    return out


def expected(truth, query, extra, tombstones=None, files=None):
    """The exact reference of one (query, extra) entry of the builders above."""
    from tests.group_reference import exact_aggregate_grouped
    if "group_ids" in extra:
        return exact_aggregate_grouped(truth, query, extra["group_ids"], extra["n_groups"], tombstones=tombstones,
                                       files=files)
    if "slide" in extra:
        from tests.sliding_reference import expand_aggregate
        return expand_aggregate(merge_truth(truth, files, query) if files is not None else truth, query, extra["slide"])
    return exact_aggregate(truth, query, tombstones=tombstones, files=files)


def two_file_arena(t0, step, seed=11):
    """Six series of two chunk files of 120 rows each on the grid t0 + k * step; file 2 starts 50 rows later, so rows
    50-119 of file 1 share file 2's times. An i64 column 1 and an f64 column 2 hold NULLs apart. -> (arena, descs,
    truth, files, merged): merged is the truth of the merged rows, built by hand (the later file wins per column when it
    holds a value: take_last_and_merge)."""
    rng = np.random.default_rng(seed)
    b = datagen.ArenaBuilder()
    truth, files, rows = {}, [], {}
    for sid in range(6):
        for f in range(2):
            n = 120
            ts = t0 + (np.arange(n, dtype=np.int64) + 50 * f) * step
            x = rng.integers(-100, 100, n).astype(np.int64)
            y = rng.random(n) * 10
            xv, yv = rng.random(n) > 0.2, rng.random(n) > 0.2
            b.add_column_group(sid, ts, [(1, cabi.TSKV_PT_I64, x, xv), (2, cabi.TSKV_PT_F64, y, yv)])
            truth.setdefault(sid, []).append((ts, {1: (x, xv), 2: (y, yv)}))
            files.append(f + 1)
            for i in range(n):
                row = rows.setdefault((sid, int(ts[i])), {})
                if xv[i]:
                    row[1] = x[i]
                if yv[i]:
                    row[2] = y[i]
    arena, descs = b.finish()
    merged = {}
    for sid in range(6):
        tss = sorted(t for s, t in rows if s == sid)
        cols = {c: (np.array([rows[(sid, t)].get(c, 0) for t in tss], dtype=dt),
                    np.array([c in rows[(sid, t)] for t in tss])) for c, dt in ((1, np.int64), (2, np.float64))}
        merged[sid] = [(np.array(tss, dtype=np.int64), cols)]
    return arena, descs, truth, np.array(files, dtype=np.uint64), merged
