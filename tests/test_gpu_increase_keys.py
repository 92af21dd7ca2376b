"""Counter increases where the records' machinery would go wrong, against tests/increase_reference.py: the records'
per-(bin, sub-bucket) offsets (rec0), the two radix sorts that read only part of each key (the slot sort's
(increase, slot) bits, the time sort's bits of the page set's time span above t_base), the grid-capped helper kernels and
the boundary stitch.

1. test_one_series_through_every_bin: series whose column groups cycle through every time codec (RLE, jittered simple8b,
   raw), value codec (narrow / wide simple8b, Gorilla, raw, run-length) and page length (short, long), added in
   shuffled descriptor order: one series' records lie in many (bin, sub) regions of rec0, and the stitch joins them.
2. test_time_key_width: one series whose pages span just under and just over 2^32 ns, about 2^62 ns, negative to
   positive times, and INT64_MIN to INT64_MAX; pages in reverse descriptor order with values whose increase changes if
   any two pages swap. Each case also runs with caller-given time bounds (tskvgpu_pages_set_time_bounds): exact ones,
   looser ones, and the whole int64 range.
3. test_tsm_file_bounds_and_value_stats: one of those page sets through a TSM file image, with its column groups' time
   bounds and its pages' value statistics set, and a predicate that prunes pages.
4. test_slot_key_width: 1-1024 selected series x 1-8 increases (mixed types, duplicates), every increase's values; the
   last slot holds the page set's earliest point and several stitched pages, among many empty records (filtered and
   all-NULL pages) before and after it in descriptor order.
5. test_scale: a generated page set with more work items of one operand than k_scan_increase has lanes, and more
   records than the helper kernels' capped grids have threads, against a vectorized reference."""
import numpy as np
import pytest

from cnosdb_b200 import cabi, datagen, tsmfile
from cnosdb_b200.engine import PushedAggregate, QueryOption
from oracle import pyoracle as orc
from tests import sweep_reference as sw
from tests.exact_arenas import add_column_group
from tests.helpers import bucket_index, bucket_spec
from tests.increase_reference import check_increase, exact_increase_cells, increase_bits, increase_cells_np

pytestmark = pytest.mark.gpu

I64, F64, U64 = cabi.TSKV_PT_I64, cabi.TSKV_PT_F64, cabi.TSKV_PT_U64
I64_MIN, I64_MAX = -2**63, 2**63 - 1
FIELDS = ((1, I64), (2, F64), (3, U64))
STEP = 1000


def inc(cid):
    return PushedAggregate(cid, dict(FIELDS)[cid], ["increase"])


def prepared(engine, pages, q, **kw):
    """-> (ScanResult, work list) of one prepared scan."""
    s = engine.prepare(pages, q, **kw)
    try:
        s.run()
        return s.finalize(), s.work_list()
    finally:
        s.close()


def check_all(res, truth, q, what, min_valid=1, **kw):
    """Every increase of `res` against the exact reference (computed once per operand column)."""
    incs = [c for c in q.columns if c.increase]
    i0 = len(res.names) - len(incs)
    n_cells = res.n_groups * res.n_buckets
    exact = {}
    for k, c in enumerate(incs):
        if c.column_id not in exact:
            exact[c.column_id] = exact_increase_cells(truth, q, c.column_id, c.phys_type, n_cells, **kw)
        check_increase(res, i0 + k, exact[c.column_id], c.phys_type, what="%s increase %d of %d" % (what, k, c.column_id))
        assert exact[c.column_id][1].sum() >= min_valid, what


# ---- 1. one series through every bin -----------------------------------------------------------------------------------
TIME_KINDS = ("rle", "s8b", "raw")
VALUE_CODECS = ("s8b_narrow", "s8b_wide", "gorilla", "raw", "rle")


def codec_for(pt, v):
    """The encoding of a column of type pt in a column group of value codec v (sweep_reference.ENCODINGS)."""
    if pt == F64:
        return "raw" if v in ("raw", "rle") else "gorilla"
    if pt == U64:
        return {"gorilla": "s8b_wide", "rle": "s8b_narrow"}.get(v, v)
    return {"gorilla": "s8b_narrow"}.get(v, v)


def every_bin_arena(seed, n_series=3):
    """n_series series, each a chain of 30 column groups: every (time codec, value codec, short / long page) once, in a
    random time order, added to the arena in a shuffled order of all series' groups."""
    rng = np.random.default_rng(seed)
    combos = [(tk, v, long) for tk in TIME_KINDS for v in VALUE_CODECS for long in (False, True)]
    groups = []
    for sid in range(n_series):
        t = sw.T0 + sid * 13
        for k in rng.permutation(len(combos)):
            tk, v, long = combos[k]
            n = int(rng.integers(sw.SHORT_PAGE_ROWS + 1, 1300)) if long else int(rng.integers(2, sw.SHORT_PAGE_ROWS + 1))
            ts = sw.timestamps(rng, tk, t, n, STEP)
            t = int(ts[-1]) + STEP * int(rng.integers(1, 4))
            groups.append((sid, ts, tk, [(c, codec_for(pt, v)) for c, pt in FIELDS], 0.1 if k % 3 == 0 else 0.0))
    a = sw.Arena()
    for g in rng.permutation(len(groups)):
        a.add(rng, *groups[g][:4], groups[g][4])
    return a.finish()


def regions_of_series(wl, descs, q):
    """{series: {column: {(bin, sub) regions holding its operand pages' work items}}}."""
    ids = [c.column_id for c in sw.scan_query(q).columns]
    out = {}
    for b in range(sw.N_BINS):
        for qc, cid in enumerate(ids):
            for sub in (0, 1):
                k = (b * len(ids) + qc) * 2 + sub
                start, fill = int(wl["region_start"][k]), int(wl["fill"][k])
                for sid in set(descs["series_id"][wl["work_page"][start:start + fill]].tolist()):
                    out.setdefault(sid, {}).setdefault(cid, set()).add((b, sub))
    return out


def test_one_series_through_every_bin(engine):
    arena, descs, truth = every_bin_arena(5)
    lo, hi = sw.span(truth)
    incs = [inc(1), inc(2), inc(3)]
    pages = engine.upload_pages(arena, descs)
    try:
        w = 37 * STEP
        fbs, nb = bucket_spec(lo, hi, w)
        q = QueryOption(incs, width=w, first_bucket_start=fbs, n_buckets=nb, group_by_series=True)
        res, wl = prepared(engine, pages, q)
        regions = regions_of_series(wl, descs, q)
        for sid in truth:
            union = set().union(*regions[sid].values())
            assert len(union) >= 8, (sid, regions[sid])
            assert len(regions[sid][1]) >= 8, (sid, sorted(regions[sid][1]))  # (i64: narrow and wide sub-buckets too)
        print("\nevery bin: (bin, sub) regions per series and column: %s" % {
            sid: {c: len(r) for c, r in v.items()} for sid, v in regions.items()})
        check_all(res, truth, q, "every bin, tumbling")
        e = sw.random_edges(np.random.default_rng(1), lo, hi, 50)
        qe = QueryOption(incs, n_buckets=e.size - 1, group_by_series=True)
        res, _ = prepared(engine, pages, qe, edges=e)
        check_all(res, truth, qe, "every bin, edges", edges=e)
        for sid in truth:
            qu = QueryOption(incs, series_ids=[sid])
            res, _ = prepared(engine, pages, qu)
            check_all(res, truth, qu, "every bin, series %d unbucketed" % sid)
    finally:
        pages.close()


# ---- 2. time-key width -------------------------------------------------------------------------------------------------
SPANS = {
    "just under 2^32": (10**12, 10**12 + 2**32 - 7),
    "just over 2^32": (10**12, 10**12 + 2**32 + 7),
    "about 2^62": (-2**50, 2**62 - 2**50 + 12345),
    "negative to positive": (-3 * 10**17, 2 * 10**17),
    "INT64_MIN to INT64_MAX": (I64_MIN, I64_MAX),
}
K_PAGES, PAGE_ROWS = 6, 40


def span_groups(lo, hi, seed):
    """K_PAGES column groups (ts, {col: (values, valid)}) of PAGE_ROWS rows STEP apart, the first starting at lo and the
    last ending at hi. Page k's values rise from a level L[k] (a permutation with noise), so the pair across each page
    boundary is a rise or a reset."""
    rng = np.random.default_rng(seed)
    span = hi - lo - (PAGE_ROWS - 1) * STEP
    starts = [lo + span * k // (K_PAGES - 1) for k in range(K_PAGES)]
    levels = rng.permutation(K_PAGES) * 1000 + rng.integers(0, 400, K_PAGES) + 500
    groups = []
    for k, s in enumerate(starts):
        ts = np.array([s + r * STEP for r in range(PAGE_ROWS)], dtype=np.int64)
        v = levels[k] + np.cumsum(rng.integers(0, 4, PAGE_ROWS))
        valid = rng.random(PAGE_ROWS) > 0.1
        valid[[0, -1]] = True
        groups.append((ts, {1: (v.astype(np.int64), valid), 2: (v + 0.25, valid), 3: (v.astype(np.uint64), valid)}))
    return groups


def page_order_matters(groups):
    """The i64 increase of the pages in time order differs from that of every order with two pages swapped."""
    pages = [cols[1][0][cols[1][1]] for _, cols in groups]
    whole = increase_bits(np.concatenate(pages), I64)[0]
    for i in range(len(pages)):
        for j in range(i + 1, len(pages)):
            p = list(pages)
            p[i], p[j] = p[j], p[i]
            if increase_bits(np.concatenate(p), I64)[0] == whole:
                return False
    return True


def span_arena(lo, hi, seed=0):
    """One series (id 7) of span_groups, from the first seed >= `seed` whose increase changes if any two pages swap
    places (a time sort that misplaces one page changes the result), added in reverse time order. -> (arena, descs,
    truth, the groups' (min, max) times in descriptor order)."""
    while not page_order_matters(span_groups(lo, hi, seed)):
        seed += 1
    groups = span_groups(lo, hi, seed)
    b = datagen.ArenaBuilder()
    for ts, cols in reversed(groups):
        b.add_column_group(7, ts, [(c, pt, cols[c][0], cols[c][1]) for c, pt in FIELDS])
    arena, descs = b.finish()
    return arena, descs, {7: groups}, [(int(ts[0]), int(ts[-1])) for ts, _ in reversed(groups)]


def span_queries(lo, hi, truth):
    """The unbucketed scan of the series, and an edge scan whose edges cut pages 1, 3 and 4 (not for a span that ends
    at INT64_MAX: its last edge would be INT64_MAX + 1)."""
    incs = [inc(1), inc(2), inc(3), inc(1)]
    out = [("unbucketed", QueryOption(incs, series_ids=[7]), {})]
    if hi < I64_MAX:
        cuts = [int(truth[7][k][0][17]) + 1 for k in (1, 3, 4)]
        e = np.array([lo] + cuts + [hi + 1], dtype=np.int64)
        out.append(("edges", QueryOption(incs, series_ids=[7], n_buckets=e.size - 1), {"edges": e}))
    return out


@pytest.mark.parametrize("name", list(SPANS))
def test_time_key_width(engine, name):
    """Upload accepts points at INT64_MIN and INT64_MAX; a span that ends at INT64_MAX runs unbucketed only. Bounds:
    none (the scan's own), exact, looser by 2^40 (clamped to int64), and the whole int64 range."""
    lo, hi = SPANS[name]
    arena, descs, truth, bounds = span_arena(lo, hi)
    queries = [(qn, q, kw, None) for qn, q, kw in span_queries(lo, hi, truth)]
    loose = [(max(I64_MIN, a - 2**40), min(I64_MAX, b + 2**40)) for a, b in bounds]
    for given, bd in (("own", None), ("exact", bounds), ("loose", loose), ("int64 range", [(I64_MIN, I64_MAX)] * len(bounds))):
        pages = engine.upload_pages(arena, descs)
        try:
            if bd is not None:
                pages.set_time_bounds(bd)
            for qn, q, kw, _ in queries:
                res, _ = prepared(engine, pages, q, **kw)
                check_all(res, truth, q, "%s, %s, bounds %s" % (name, qn, given), **kw)
        finally:
            pages.close()


def test_tsm_file_bounds_and_value_stats(engine):
    """The 2^62 page set written to a TSM file image and loaded back: the scan takes the file's column-group bounds and
    page statistics, and a predicate on column 1 prunes the pages whose maximum lies below it."""
    from tests.test_tsm_file import page_value_stats
    lo, hi = SPANS["about 2^62"]
    arena, descs, truth, bounds = span_arena(lo, hi, seed=3)
    f = tsmfile.load(tsmfile.write(arena, descs, np.array(bounds, dtype=np.int64), value_stats=page_value_stats(arena, descs)))
    assert (f.cg_bounds == np.array(bounds)).all()
    pages = engine.upload_pages(f.arena, f.descs)
    try:
        pages.set_time_bounds(f.cg_bounds)
        pages.set_value_stats(f.value_stats)
        q = QueryOption([inc(1), inc(2), inc(3)], series_ids=[7], predicates=[(1, I64, ">=", 2500)])
        res, _ = prepared(engine, pages, q)
        assert engine.counters()["pruned_page_count"] > 0
        check_all(res, truth, q, "TSM file, pruned")
        e = np.array([lo, 0, 2**61, hi + 1], dtype=np.int64)
        qe = QueryOption([inc(3), inc(1)], series_ids=[7], n_buckets=3, predicates=[(2, F64, "<", 4000.0)])
        res, _ = prepared(engine, pages, qe, edges=e)
        check_all(res, truth, qe, "TSM file, edges", edges=e)
    finally:
        pages.close()


# ---- 4. slot-key width -------------------------------------------------------------------------------------------------
SLOT_COUNTS = (1, 2, 3, 4, 8, 64, 1024)
INC_COUNTS = (1, 2, 3, 4, 8)
INC_COLS = (1, 2, 3, 3, 1, 2, 1, 3)
FILTER = 4  # an i64 column the query's predicate keeps at >= 0: -1 in the filtered pages


def slot_arena(n_slots, seed):
    """n_slots series (ids 3 + 5 * slot); the last one holds the page set's earliest point and five column groups whose
    boundaries are rises and resets; the others one or two short groups later on. Empty records: column groups whose
    rows the predicate filters (behind jittered and regular time), and column groups whose operands are all NULL, of
    series before and after the last one in descriptor order."""
    rng = np.random.default_rng([n_slots, seed])
    sids = [3 + 5 * s for s in range(n_slots)]
    t_late = sw.T0 + 1000 * STEP
    groups = []  # (descriptor-order key, sid, ts, time kind, {col: (values, valid)})

    def group(sid, ts, kind, level, mode, key):
        n = len(ts)
        v = level + np.cumsum(rng.integers(0, 5, n))
        ok = np.zeros(n, dtype=bool) if mode == "null" else rng.random(n) > 0.1
        cols = {1: (v.astype(np.int64), ok), 2: (v + 0.5, ok.copy()), 3: (v.astype(np.uint64), ok.copy()),
                FILTER: (np.full(n, -1 if mode == "filtered" else 1, dtype=np.int64), np.ones(n, dtype=bool))}
        if mode == "first":
            for c in (1, 2, 3):
                cols[c][1][0] = True  # (the earliest point is selected: time key 0)
        groups.append((key, sid, np.asarray(ts, dtype=np.int64), kind, cols))

    last = sids[-1]
    t = sw.T0
    for k, lv in enumerate(rng.permutation(5) * 1000 + 100):
        n = int(rng.integers(20, 40))
        group(last, t + np.arange(n) * STEP, "rle", lv, "first" if k == 0 else "real", (len(sids), 4 - k))
        t += (n + 2) * STEP
    for k in range(3):  # empty groups of the last series, after its data
        n = int(rng.integers(5, 30))
        ts = sw.timestamps(rng, ("s8b", "rle", "rle")[k], t, n, STEP)
        group(last, ts, ("s8b", "rle", "rle")[k], 0, ("filtered", "filtered", "null")[k], (len(sids), 5 + k) if k else (-1, k))
        t = int(ts[-1]) + 2 * STEP
    others = sids[:-1]
    for j, sid in enumerate(others):
        tt = t_late + int(rng.integers(0, 50)) * STEP
        for g in range(2 if n_slots <= 64 else 1):
            n = int(rng.integers(3, 10))
            group(sid, tt + np.arange(n) * STEP, "rle", int(rng.integers(0, 10**6)), "real", (j, g))
            tt += (n + 1) * STEP
    for j in range(12):  # empty groups of other series (or of the last one, with one series), before and after it
        sid = others[int(rng.integers(0, len(others)))] if others else last
        kind = ("s8b", "rle", "raw")[j % 3]
        mode = "null" if j % 4 == 3 else "filtered"
        ts = sw.timestamps(rng, kind, t_late + (1000 + 100 * j) * STEP, int(rng.integers(3, 40)), STEP)
        group(sid, ts, kind, 0, mode, (-1 if j % 2 else len(sids) + 1, 10 + j))
    b = datagen.ArenaBuilder()
    truth = {}
    for _, sid, ts, kind, cols in sorted(groups, key=lambda g: g[0]):
        fields = [(c, I64 if c == FILTER else dict(FIELDS)[c], v, ok) for c, (v, ok) in cols.items()]
        add_column_group(b, sid, ts, fields, raw_time=kind == "raw")
        truth.setdefault(sid, []).append((ts, cols))
    arena, descs = b.finish()
    return arena, descs, truth, sids


@pytest.mark.parametrize("n_slots", SLOT_COUNTS)
def test_slot_key_width(engine, n_slots):
    """Every n_increases of INC_COUNTS over the same page set; with n_slots and n_increases powers of two the top
    increase's last slot has every bit of the slot sort's key set but one (an empty record's key has all)."""
    arena, descs, truth, sids = slot_arena(n_slots, 1)
    pages = engine.upload_pages(arena, descs)
    try:
        for n_inc in INC_COUNTS:
            s0 = SLOT_COUNTS.index(n_slots)
            cols = [inc(INC_COLS[(s0 + k) % len(INC_COLS)]) for k in range(n_inc)]
            q = QueryOption(cols, series_ids=np.array(sids, dtype=np.uint32), group_by_series=True,
                            predicates=[(FILTER, I64, ">=", 0)])
            res, _ = prepared(engine, pages, q)
            what = "%d slots, %d increases" % (n_slots, n_inc)
            check_all(res, truth, q, what, min_valid=n_slots)
            # the last slot's increase holds every stitch of its five pages
            for k, c in enumerate(cols):
                v, ok = res.values[len(res.names) - n_inc + k], res.validity[len(res.names) - n_inc + k]
                assert ok[n_slots - 1] and v[n_slots - 1] != 0, what
    finally:
        pages.close()


# ---- 5. scale ----------------------------------------------------------------------------------------------------------
SCALE_SERIES, SCALE_CHUNKS, SCALE_ROWS = 120_000, 7, 4
STITCH_THREADS = 4096 * 256  # k_increase_init / _gather / _stitch: grid capped at 4096 blocks of 256


def scale_arena():
    """SCALE_CHUNKS generated page sets of the same series, one after the other in time (datagen MIXED: even series
    hold i64 column 1, odd series f64 column 2; NULL rows in 10% of the pages), concatenated."""
    parts, ds, off = [], [], 0
    for k in range(SCALE_CHUNKS):
        g = datagen.generate(SCALE_SERIES, n_fields=1, n_points=SCALE_ROWS, value_kind=datagen.MIXED, seed=11 + k,
                             t0=sw.T0 + k * SCALE_ROWS * STEP, step=STEP, null_page_permille=100, null_row_permille=200)
        d = g.descs.copy()
        d["offset"] += off
        pad = (-g.arena.size) % 4096
        parts += [g.arena.copy(), np.zeros(pad, dtype=np.uint8)]
        off += g.arena.size + pad
        ds.append(d)
        g.close()
    return np.concatenate(parts), np.concatenate(ds)


def test_scale(engine):
    import torch
    lanes = torch.cuda.get_device_properties(engine.device).multi_processor_count * 16 * 128
    arena, descs = scale_arena()
    w = 5 * STEP
    lo, hi = sw.T0, sw.T0 + SCALE_CHUNKS * SCALE_ROWS * STEP
    fbs, nb = bucket_spec(lo, hi, w)
    cols = [inc(1), PushedAggregate(2, F64, ["increase"]), inc(1), PushedAggregate(2, F64, ["increase"])]
    q = QueryOption(cols, width=w, first_bucket_start=fbs, n_buckets=nb, group_by_series=True)
    pages = engine.upload_pages(arena, descs)
    try:
        res, wl = prepared(engine, pages, q)
    finally:
        pages.close()
    # the work list: one operand's region holds more items than k_scan_increase has lanes, and the records of all
    # increases outnumber the helper kernels' threads
    fill = wl["fill"].astype(np.int64).reshape(sw.N_BINS, 2, 2)
    assert fill[:, 0].max() > 1.25 * lanes and fill[:, 1].max() > 1.25 * lanes, (fill[:, :, :].max(), lanes)
    records = 2 * int(fill[:, 0].sum()) + 2 * int(fill[:, 1].sum())
    assert records > 1.4 * STITCH_THREADS, records
    assert res.n_groups == SCALE_SERIES and int(res.n_groups).bit_length() == 17
    print("\nscale: %d lanes, largest operand regions %d / %d items, %d records" % (
        lanes, fill[:, 0].max(), fill[:, 1].max(), records))
    # the reference: every page decoded by the CPU checker, each field page behind the time page before it
    dec = orc.decode_pages(arena, descs)
    vals = np.stack([v for v, _ in dec])
    valid = np.stack([m for _, m in dec])
    slot_of = {int(s): i for i, s in enumerate(np.unique(descs["series_id"]))}
    n_cells = res.n_groups * res.n_buckets
    for k, c in enumerate(cols):
        field = np.nonzero(descs["column_id"] == c.column_id)[0]
        tp = field - 1
        assert (descs["phys_type"][tp] == cabi.TSKV_PT_TIME).all() and (descs["series_id"][tp] == descs["series_id"][field]).all()
        t = vals[tp].view(np.int64).ravel()
        ok = (valid[field] & valid[tp]).ravel()
        slots = np.repeat(np.array([slot_of[int(s)] for s in descs["series_id"][field]]), SCALE_ROWS)
        b, in_b = bucket_index(t, q)
        ok &= in_b
        exact = increase_cells_np(slots[ok] * nb + b[ok], t[ok], vals[field].ravel()[ok], c.phys_type, n_cells)
        check_increase(res, len(res.names) - len(cols) + k, exact, c.phys_type, what="scale increase %d" % k)
        assert exact[1].sum() > SCALE_SERIES, k
