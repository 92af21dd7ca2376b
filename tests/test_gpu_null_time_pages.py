"""Time pages with NULL rows through the fused scan against the oracle, which restates is_not_null(time)
(transform_time_window.rs:313): a NULL-time row is dropped, a NULL row 0 of a simple8b time page swallows the first
timestamp (timestamp.rs:273-279), an all-NULL time page holds no row. Time pages that would be RLE, jittered simple8b
and raw, with NULLs at row 0, across the 31 / 32 / 33 bitmap-word edges, at the last row, everywhere and at random;
zig-zag simple8b i64 / u64, Gorilla f64, raw i64 and boolean values with NULLs on and next to the NULL-time rows.
Every query runs GROUP BY bucket, series, tags and unbucketed, with and without FIRST / LAST; the scan's
points_decoded and rows_in_range are checked against counts restated from the generated arrays. Column pairs and
medians, whose passes decode the same pages row by row with their own NULL-time handling, are held to their exact
references over the rows with a valid timestamp."""
import functools
from types import SimpleNamespace

import numpy as np
import pytest

from cnosdb_b200 import cabi, datagen
from cnosdb_b200.engine import PushedAggregate, QueryOption, TskvError
from oracle import pyoracle as orc
from tests.covariance_reference import check_pair, exact_pair_cells
from tests.helpers import assert_results_equal, bucket_spec, make_query
from tests.median_reference import check_median, exact_median_cells

pytestmark = pytest.mark.gpu

T0, STEP, W = 10**12, 1000, 7_000
KINDS = ("rle", "s8b", "raw")
PATTERNS = ("row0", "lead", "edges", "last", "all", "zero", "random", "none")
LENGTHS = (40, 66, 97, 130)
FIELDS = ((1, cabi.TSKV_PT_I64), (2, cabi.TSKV_PT_F64), (3, cabi.TSKV_PT_U64), (4, cabi.TSKV_PT_I64),
          (5, cabi.TSKV_PT_BOOL))
PLAIN = ("count", "sum", "min", "max", "mean")
SEL = ("count", "min", "max", "first", "last")


def time_validity(pattern, n, rng):
    tv = np.ones(n, dtype=bool)
    if pattern == "row0":
        tv[0] = False
    elif pattern == "lead":  # a leading run across the first bitmap-word edge
        tv[:33] = False
    elif pattern == "edges":  # runs across the bitmap-word edges
        for a, b in ((31, 34), (63, 66), (95, 97)):
            tv[a:b] = False
    elif pattern == "last":
        tv[-1] = False
    elif pattern in ("all", "zero"):
        tv[:] = False
    elif pattern == "random":
        tv = rng.random(n) >= 0.3
    return tv


def add_group(b, sid, kind, ts, tv, fields, tvals=None):
    """The time page as the writer encodes it (RLE for the grid, simple8b for jitter), or raw; it holds `tvals` (default:
    the valid rows' timestamps). A NULL row 0 of a simple8b time page swallows the page's first value: such a page holds
    one more value, in front."""
    n = len(ts)
    tvals = ts[tv] if tvals is None else tvals
    if kind == "s8b" and not tv[0] and tv.any():
        tvals = np.concatenate([tvals[:1] - 500, tvals])
    tenc = datagen.encode_raw if kind == "raw" else datagen.encode_timestamps
    b.add_page(datagen.build_page(tenc(tvals), n, tv), sid, 0, cabi.TSKV_PT_TIME, n)
    for col, pt, vals, valid, *enc in fields:
        enc = enc[0] if enc else (datagen.encode_floats if pt == cabi.TSKV_PT_F64 else
                                  datagen.encode_bools if pt == cabi.TSKV_PT_BOOL else datagen.encode_integers)
        kept = vals[valid]
        if pt == cabi.TSKV_PT_U64 and enc is datagen.encode_integers:
            kept = kept.view(np.int64)
        b.add_page(datagen.build_page(enc(kept), n, valid), sid, col, pt, n)


@functools.lru_cache(maxsize=None)
def null_time_arena():
    """One column group per series; series sid has time kind KINDS[sid % 3] and NULL pattern PATTERNS[sid // 3 % 8].
    The valid rows carry the timestamps (the grid, or the grid with jitter), so an RLE page stays RLE. "all" time
    pages are empty (DK_ALLNULL: no rows), "zero" ones hold timestamps behind an all-zero bitmap (rows that all fail
    is_not_null(time), whose values are still decoded). Returns (arena, descs, truth) with truth[sid] = (timestamps,
    time validity, {column: value validity}, whether the time page is empty, {column: values})."""
    rng = np.random.default_rng(31)
    b = datagen.ArenaBuilder()
    truth = {}
    for sid in range(48):
        kind, pattern = KINDS[sid % 3], PATTERNS[sid // 3 % 8]
        n = LENGTHS[sid % 4]
        tv = time_validity(pattern, n, rng)
        k = np.cumsum(tv) - 1  # index of each valid row among the valid rows
        ts = T0 + (sid % 5) * 300 + k * STEP + (rng.integers(-300, 301, n) if kind == "s8b" else 0)
        ts = np.where(tv, ts, 0).astype(np.int64)
        fl, cols, values = [], {}, {}
        for col, pt in FIELDS:
            valid = rng.random(n) >= 0.15
            valid[~tv] = rng.random(int((~tv).sum())) < 0.5  # values on NULL-time rows, and NULLs next to them
            valid[1:][~tv[:-1]] &= rng.random(int((~tv[:-1]).sum())) < 0.5
            if pt == cabi.TSKV_PT_F64:
                v = np.cumsum(rng.integers(-3, 4, n)) + rng.random(n)
            elif pt == cabi.TSKV_PT_U64:
                v = rng.integers(0, 2**63, n, dtype=np.uint64) + np.uint64(sid % 2) * np.uint64(2**63)
            elif pt == cabi.TSKV_PT_BOOL:
                v = rng.random(n) < 0.5
            else:
                v = np.cumsum(rng.integers(-50, 51, n)).astype(np.int64)
            fl.append((col, pt, v, valid) + ((datagen.encode_raw,) if col == 4 else ()))
            cols[col] = valid
            values[col] = v
        tvals = T0 + np.arange(n, dtype=np.int64) * STEP if pattern == "zero" else None
        add_group(b, sid, kind, ts, tv, fl, tvals)
        truth[sid] = (ts, tv, cols, pattern == "all", values)
    arena, descs = b.finish()
    return arena, descs, truth


def grouped_oracle(arena, descs, q, group_ids, n_groups, tombs):
    """GROUP BY tags from the oracle: group g's cells are the GROUP BY bucket scan of g's members."""
    parts = []
    for g in range(n_groups):
        sub = QueryOption(q.columns, series_ids=q.series_ids[group_ids == g], time_ranges=q.time_ranges,
                          predicates=q.predicates, width=q.width, first_bucket_start=q.first_bucket_start,
                          n_buckets=q.n_buckets)
        parts.append(orc.scan_aggregate(arena, descs, sub, tombstones=tombs))
    return SimpleNamespace(names=parts[0].names, phys=parts[0].phys, values=np.concatenate([p.values for p in parts], axis=1),
                           validity=np.concatenate([p.validity for p in parts], axis=1))


def expected_counts(truth, q, sel):
    """(points_decoded, rows_in_range) restated from the arrays; queries without predicates or tombstones."""
    points = rows = 0
    for sid in sel:
        ts, tv, cols, empty, _ = truth[int(sid)]
        if empty:  # an empty (DK_ALLNULL) time page holds no row: nothing is decoded
            continue
        inr = tv.copy()
        if q.time_ranges:
            inr &= np.any([(ts >= lo) & (ts <= hi) for lo, hi in q.time_ranges], axis=0)
            if not inr.any():  # the column group's time range meets no query range: statistics pruning
                continue
        for c in q.columns:
            points += int(cols[c.column_id].sum())
            rows += int(inr.sum())
    return points, rows


def queries(sids):
    t_hi = T0 + 140 * STEP
    fbs, nb = bucket_spec(T0 - 1000, t_hi, W)
    grid = dict(width=W, first_bucket_start=fbs, n_buckets=nb)
    ranges = ([], [(T0 + 5 * STEP, T0 + 90 * STEP)], [(T0, T0 + 31 * STEP), (T0 + 33 * STEP + 1, T0 + 64 * STEP), (T0 + 100 * STEP, t_hi)])
    for aggs in (PLAIN, SEL):
        fields = FIELDS[:4] if aggs is PLAIN else FIELDS
        for r in ranges:
            for by in ("bucket", "series", "tags", "none"):
                kw = dict(grid, group_by_series=by == "series") if by != "none" else {}
                yield by, make_query(fields, aggs=aggs, series_ids=sids, time_ranges=r, **kw)
        yield "predicate", make_query(fields, aggs=aggs, series_ids=sids[::2], time_ranges=ranges[1],
                                      predicates=[(1, cabi.TSKV_PT_I64, ">", -40)], **grid)


def tombstones(sids):
    out = [(None, None, T0 + 70 * STEP, T0 + 72 * STEP)]
    for sid in sids[::3]:
        out.append((sid, None, T0 + 20 * STEP - 100, T0 + 33 * STEP))
    for sid in sids[1::3]:
        out.append((sid, 2, T0 + 30 * STEP, T0 + 65 * STEP))
        out.append((sid, 5, T0, T0 + 3 * STEP))
    return cabi.tombstones(out)


def check(engine, pages, arena, descs, q, by, tombs, what):
    group_ids = n_groups = None
    if by == "tags":
        group_ids = (np.arange(q.series_ids.size) * 7 % 4).astype(np.uint32)
        n_groups = 4
        exp = grouped_oracle(arena, descs, q, group_ids, n_groups, tombs)
    else:
        exp = orc.scan_aggregate(arena, descs, q, tombstones=tombs)
    got = engine.scan_aggregate(pages, q, group_ids=group_ids, n_groups=n_groups)
    assert_results_equal(got, exp, what=what)


def test_null_time_rows_match_the_oracle(engine):
    arena, descs, truth = null_time_arena()
    pages = engine.upload_pages(arena, descs)
    sids = np.array(sorted(truth), dtype=np.uint32)
    for by, q in queries(sids):
        what = "%s ranges=%s aggs=%#x" % (by, q.time_ranges, q.columns[0].agg_mask)
        check(engine, pages, arena, descs, q, by, None, what)
        if not q.predicates:
            c = engine.counters()
            assert (c["points_decoded"], c["rows_in_range"]) == expected_counts(truth, q, q.series_ids), what
    # Tombstones: the reference binary-searches the page's raw time buffer, in which a NULL row reads as 0
    # (update_nullbits_by_time_range, tsm/reader.rs:634-656), and the scan tests every row's own timestamp. The two
    # agree while that buffer stays sorted - NULL rows only in front of the first valid one - so these queries select
    # those series.
    sids = np.array([sid for sid, (ts, *_) in sorted(truth.items()) if (np.diff(ts) >= 0).all()], dtype=np.uint32)
    tombs = tombstones(sids)
    pages.set_tombstones(tombs)
    for by, q in queries(sids):
        check(engine, pages, arena, descs, q, by, tombs, "tombstones " + by)
    pages.close()


def test_null_time_rows_pairs_and_medians(engine):
    """Pairs and medians over every series of the arena, by series and bucket: their passes must drop the NULL-time
    rows (and, behind a simple8b time page with a NULL row 0, the swallowed first timestamp) as the fused scan does. The
    exact references read the rows with a valid timestamp."""
    arena, descs, truth = null_time_arena()
    rows = {sid: [(ts[tv], {c: (values[c][tv], cols[c][tv]) for c, _ in FIELDS})]
            for sid, (ts, tv, cols, _, values) in truth.items()}
    num = [(c, pt) for c, pt in FIELDS if pt != cabi.TSKV_PT_BOOL]
    # every numeric column is x once with the next one and once with itself (the pair passes walk x's pages)
    pairs = [x + num[(i + 1) % len(num)] for i, x in enumerate(num)] + [x + x for x in num]
    fbs, nb = bucket_spec(T0 - 1000, T0 + 140 * STEP, W)
    q = QueryOption([PushedAggregate(c, pt, ["median"]) for c, pt in num],
                    series_ids=np.array(sorted(truth), dtype=np.uint32), width=W, first_bucket_start=fbs, n_buckets=nb,
                    group_by_series=True, pairs=pairs)
    pages = engine.upload_pages(arena, descs)
    try:
        got = engine.scan_aggregate(pages, q)
    finally:
        pages.close()
    n_cells = got.n_groups * got.n_buckets
    for k, p in enumerate(pairs):
        check_pair(got, k, exact_pair_cells(rows, q, p, n_cells), what="NULL-time rows pair %s" % (p,))
    for k, (c, pt) in enumerate(num):
        check_median(got, len(got.names) - len(num) + k, exact_median_cells(rows, q, c, pt, n_cells),
                     what="NULL-time rows median of %d" % c)


@pytest.mark.parametrize("kind", ["raw", "s8b", "s8b_row0"])
def test_time_page_with_more_valid_bits_than_values(engine, kind):
    """A time page (NULLs at rows 3 and 40) whose validity bitmap announces more timestamps than its data holds;
    s8b_row0: NULL row 0 and as many values as valid rows, one too few once row 0 has swallowed the first."""
    n = 100
    tv = np.ones(n, dtype=bool)
    tv[[0] if kind == "s8b_row0" else [3, 40]] = False
    ts = T0 + np.arange(n, dtype=np.int64) * STEP + (np.arange(n) * 37 % 300 if kind != "raw" else 0)
    short = ts[tv][: {"raw": -5, "s8b": 60, "s8b_row0": None}[kind]]
    enc = datagen.encode_raw if kind == "raw" else datagen.encode_timestamps
    b = datagen.ArenaBuilder()
    b.add_column_group(1, ts[tv], [(1, cabi.TSKV_PT_I64, np.arange(int(tv.sum())), None)])  # a sound group first
    tpage = len(b.descs)
    b.add_page(datagen.build_page(enc(short), n, tv), 2, 0, cabi.TSKV_PT_TIME, n)
    b.add_page(datagen.build_page(datagen.encode_integers(np.arange(n, dtype=np.int64)), n), 2, 1, cabi.TSKV_PT_I64, n)
    arena, descs = b.finish()
    fbs, nb = bucket_spec(T0, T0 + n * STEP, W)
    pages = engine.upload_pages(arena, descs)
    for aggs in (PLAIN, SEL):
        q = make_query([(1, cabi.TSKV_PT_I64)], aggs=aggs, width=W, first_bucket_start=fbs, n_buckets=nb)
        with pytest.raises(orc.OracleError) as oe:
            orc.scan_aggregate(arena, descs, q)
        with pytest.raises(TskvError) as ge:
            engine.scan_aggregate(pages, q)
        assert oe.value.status == ge.value.status == cabi.TSKV_ERR_BITSET_MISMATCH
        assert ge.value.page == tpage
    pages.close()
