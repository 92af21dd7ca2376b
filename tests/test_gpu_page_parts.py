"""Pages cut at restart points (cnosdb_b200/csrc/skip_kernels.cuh): a scan that enters every simple8b / gorilla page at
several rows at once must give exactly what the oracle (which, like the reference, decodes every page from its first
byte) gives - for every number of parts, with nulls, jitter, time ranges, tombstones, row filters, long pages and
malformed streams."""
import numpy as np
import pytest

from cnosdb_b200 import cabi, datagen
from cnosdb_b200.engine import PushedAggregate, QueryOption, TskvError
from oracle import pyoracle as orc
from tests.helpers import assert_results_equal, bucket_spec, make_query, random_arena
from tests.test_gpu_parity import random_tombstones

pytestmark = pytest.mark.gpu

AGGS = ("count", "sum", "min", "max", "mean")  # FIRST / LAST scans never cut pages
FIELDS = ((1, cabi.TSKV_PT_I64), (2, cabi.TSKV_PT_F64), (3, cabi.TSKV_PT_U64))
PARTS = ["1", "2", "3", "8", "auto"]


def set_parts(monkeypatch, parts):
    if parts == "auto":
        monkeypatch.delenv("TSKV_PARTS", raising=False)
    else:
        monkeypatch.setenv("TSKV_PARTS", parts)


@pytest.mark.parametrize("parts", PARTS)
def test_c4_shape_cut_into_parts(engine, parts, monkeypatch):
    set_parts(monkeypatch, parts)
    g = datagen.generate(3000, n_fields=2, n_points=1000, value_kind=datagen.MIXED, seed=40, jitter_permille=300,
                         jitter_max=999_999, null_page_permille=200, null_row_permille=80)
    pages = engine.upload_pages(g.arena, g.descs)
    w = 60_000_000_000
    fbs, nb = bucket_spec(datagen.TSBS_T0 - 1_000_000, datagen.TSBS_T0 + 999 * datagen.TSBS_STEP + 1_000_000, w)
    sel = np.arange(0, 3000, 3, dtype=np.uint32)
    cols = [PushedAggregate(c, cabi.TSKV_PT_I64, AGGS) for c in (1, 2)] + [PushedAggregate(c, cabi.TSKV_PT_F64, AGGS) for c in (3, 4)]
    t0, st = datagen.TSBS_T0, datagen.TSBS_STEP
    for ranges in ([], [(t0 + 130 * st + 1, t0 + 777 * st)], [(t0 + 5 * st, t0 + 100 * st), (t0 + 250 * st, t0 + 260 * st), (t0 + 900 * st, t0 + 2000 * st)]):
        for gbs in (False, True):
            q = QueryOption(cols, series_ids=sel, time_ranges=ranges, width=w, first_bucket_start=fbs, n_buckets=nb, group_by_series=gbs)
            got = engine.scan_aggregate(pages, q)
            exp, pts = orc.scan_aggregate(g.arena, g.descs, q, n_threads=8, return_points=True)
            assert_results_equal(got, exp, what="parts=%s ranges=%s gbs=%s" % (parts, ranges, gbs))
            assert engine.counters()["points_decoded"] == pts
    q = QueryOption(cols, series_ids=sel, time_ranges=[(t0 + 300 * st, t0 + 301 * st)])  # unbucketed
    assert_results_equal(engine.scan_aggregate(pages, q), orc.scan_aggregate(g.arena, g.descs, q, n_threads=8), what="unbucketed")
    pages.close()


@pytest.mark.parametrize("parts", ["2", "8", "auto"])
@pytest.mark.parametrize("variant", ["nulls", "jitter", "multi_cg", "raw"])
def test_random_pages_tombstones_and_row_filters_cut_into_parts(engine, variant, parts, monkeypatch):
    set_parts(monkeypatch, parts)
    rng = np.random.default_rng(77 + len(variant))
    kw = dict(n_series=60, n_points=700, fields=FIELDS, null_frac=0.25)
    if variant == "jitter":
        kw.update(jitter=300, null_frac=0.02)
    if variant == "multi_cg":
        kw.update(multi_cg=True, null_frac=0.05)
    if variant == "raw":
        kw["raw_frac"] = 0.4
    arena, descs, _ = random_arena(rng, **kw)
    pages = engine.upload_pages(arena, descs)
    t_lo, t_hi = 1_000_000 - 400, 1_000_000 + 1_500_000
    fbs, nb = bucket_spec(t_lo, t_hi, 17_000, origin=3)
    sel = np.array(sorted(rng.choice(np.arange(60), 40, replace=False)), dtype=np.uint32)
    preds = [(1, cabi.TSKV_PT_I64, ">", -20), (2, cabi.TSKV_PT_F64, "<=", 9.5)]
    for gbs in (False, True):
        for ranges in ([], [(t_lo + 130_000, t_lo + 131_000), (t_lo + 300_500, t_lo + 655_000)]):
            for p in ([], preds):
                q = make_query(FIELDS, aggs=AGGS, series_ids=sel, time_ranges=ranges, origin=3, width=17_000, first_bucket_start=fbs,
                               n_buckets=nb, group_by_series=gbs, predicates=p)
                assert_results_equal(engine.scan_aggregate(pages, q), orc.scan_aggregate(arena, descs, q),
                                     what="%s parts=%s gbs=%s %s %s" % (variant, parts, gbs, ranges, p))
    tombs = random_tombstones(rng, descs, t_lo, 1_000_000 + 700_000)
    pages.set_tombstones(tombs)
    for gbs in (False, True):
        q = make_query(FIELDS, aggs=AGGS, series_ids=sel, time_ranges=[(t_lo + 30_000, t_lo + 650_000)], origin=3, width=17_000,
                       first_bucket_start=fbs, n_buckets=nb, group_by_series=gbs)
        assert_results_equal(engine.scan_aggregate(pages, q), orc.scan_aggregate(arena, descs, q, tombstones=tombs), what="tombstones")
    pages.close()


@pytest.mark.parametrize("parts", ["4", "64", "auto"])
def test_long_pages_and_mixed_lengths(engine, parts, monkeypatch):
    """Pages of 1 .. 50 000 rows in one bin: short pages have fewer parts than the bin's launch (idle lanes), the long
    ones are cut into up to 64 parts."""
    set_parts(monkeypatch, parts)
    rng = np.random.default_rng(5)
    b = datagen.ArenaBuilder()
    lens = [1, 127, 128, 129, 255, 256, 257, 1000, 4097, 50_000, 128 * 40, 128 * 40 + 1]
    for sid, n in enumerate(lens * 3):
        ts = 10_000 + np.arange(n, dtype=np.int64) * 1000 + (rng.integers(-300, 301, n) if sid % 2 else 0)
        valid = rng.random(n) > 0.1 if sid % 3 == 0 else None
        b.add_column_group(sid, ts, [(1, cabi.TSKV_PT_I64, np.cumsum(rng.integers(-9, 10, n)), valid),
                                     (2, cabi.TSKV_PT_F64, np.cumsum(rng.integers(-3, 4, n)) + rng.random(n), valid)])
    arena, descs = b.finish()
    pages = engine.upload_pages(arena, descs)
    fbs, nb = bucket_spec(0, 10_000 + 50_001 * 1000, 250_000)
    for gbs in (False, True):
        for ranges in ([], [(10_000 + 128_000, 10_000 + 3_000_500)]):
            q = make_query(FIELDS[:2], aggs=AGGS, time_ranges=ranges, width=250_000, first_bucket_start=fbs, n_buckets=nb, group_by_series=gbs)
            got = engine.scan_aggregate(pages, q)
            exp, pts = orc.scan_aggregate(arena, descs, q, return_points=True)
            assert_results_equal(got, exp, what="lengths parts=%s gbs=%s %s" % (parts, gbs, ranges))
            assert engine.counters()["points_decoded"] == pts
    pages.close()


@pytest.mark.parametrize("case,status", [("extra_values", 0), ("early_sentinel", cabi.TSKV_ERR_BITSET_MISMATCH),
                                         ("truncated_tail", cabi.TSKV_ERR_SHORT_BLOCK), ("truncated_middle", cabi.TSKV_ERR_SHORT_BLOCK),
                                         ("short_simple8b", cabi.TSKV_ERR_BITSET_MISMATCH)])
def test_malformed_streams_report_the_reference_errors_when_cut(engine, case, status, monkeypatch):
    """A stream that breaks before its last restart point gets no restart points (decoded whole, error and all); one
    that breaks after it is caught by the lane of the last part."""
    monkeypatch.setenv("TSKV_PARTS", "8")
    n = 1000
    vals = np.cumsum(np.arange(n) % 5).astype(np.float64) * 0.37 + 1.5
    ivals = np.cumsum(np.arange(n) % 7 - 3).astype(np.int64)
    ts = datagen.TSBS_T0 + np.arange(n, dtype=np.int64) * datagen.TSBS_STEP
    b = datagen.ArenaBuilder()
    b.add_page(datagen.build_page(datagen.encode_timestamps(ts), n), 5, 0, cabi.TSKV_PT_TIME, n)
    pt = cabi.TSKV_PT_F64
    if case == "extra_values":
        data = datagen.encode_floats(np.concatenate([vals, np.arange(30) * 3.25]))
    elif case == "early_sentinel":
        data = datagen.encode_floats(vals[:700])
    elif case == "truncated_tail":
        data = datagen.encode_floats(vals)[:-24]
    elif case == "truncated_middle":
        data = datagen.encode_floats(vals)[:600]
    else:
        pt = cabi.TSKV_PT_I64
        data = datagen.encode_integers(ivals[:520])
    b.add_page(datagen.build_page(data, n), 5, 1, pt, n)
    b.add_column_group(6, ts, [(1, pt, np.arange(n) * (0.5 if pt == cabi.TSKV_PT_F64 else 2), None)])
    arena, descs = b.finish()
    w = 60_000_000_000
    fbs, nb = bucket_spec(datagen.TSBS_T0, datagen.TSBS_T0 + 999 * datagen.TSBS_STEP, w)
    q = QueryOption([PushedAggregate(1, pt, AGGS)], width=w, first_bucket_start=fbs, n_buckets=nb)
    pages = engine.upload_pages(arena, descs)
    if status == 0:
        assert_results_equal(engine.scan_aggregate(pages, q), orc.scan_aggregate(arena, descs, q), what=case)
    else:
        with pytest.raises(orc.OracleError) as oe:
            orc.scan_aggregate(arena, descs, q)
        assert oe.value.status == status
        with pytest.raises(TskvError) as ge:
            engine.scan_aggregate(pages, q)
        assert ge.value.status == status and ge.value.page == 1
    pages.close()


def test_cut_and_whole_scans_agree_bit_for_bit_on_integers(engine, monkeypatch):
    """Size-independent property at a size the oracle is not run on: every number of parts gives the same integer
    aggregates and the same decoded-point count as the uncut scan."""
    g = datagen.generate(40_000, n_fields=1, n_points=1000, value_kind=datagen.MIXED, seed=9, jitter_permille=200, jitter_max=999_999,
                         null_page_permille=10, null_row_permille=50)
    pages = engine.upload_pages(g.arena, g.descs)
    w = 60_000_000_000
    fbs, nb = bucket_spec(datagen.TSBS_T0 - 1_000_000, datagen.TSBS_T0 + 999 * datagen.TSBS_STEP + 1_000_000, w)
    cols = [PushedAggregate(1, cabi.TSKV_PT_I64, AGGS), PushedAggregate(2, cabi.TSKV_PT_F64, ("count", "min", "max"))]
    q = QueryOption(cols, width=w, first_bucket_start=fbs, n_buckets=nb)
    ref, ref_pts = None, None
    for parts in ("1", "2", "4", "8"):
        monkeypatch.setenv("TSKV_PARTS", parts)
        r = engine.scan_aggregate(pages, q)
        pts = engine.counters()["points_decoded"]
        if ref is None:
            ref, ref_pts = r, pts
            continue
        assert pts == ref_pts
        for j in range(len(r.names)):
            assert (r.validity[j] == ref.validity[j]).all()
            if r.names[j][1] != "mean":
                assert (r.values[j] == ref.values[j]).all(), (parts, r.names[j])
    pages.close()


def expected_reads(descs, truth, qcols, sel=None, ranges=(), preds=()):
    """(page_read_count, page_read_bytes, pruned_page_count) restated from the generated arrays. Per column group of a
    selected series: its pages of the query columns `qcols` are pruned when its [min_ts, max_ts] meets none of the time
    ranges, or when one predicate's page in the group has no non-null value that satisfies the comparison (predicates
    with <, <=, > or >=, whose truth on [min, max] is decided at an end); otherwise they are read, with the group's time
    page once. truth lists the column groups in descriptor order (ArenaBuilder order)."""
    ops = {"<": np.less, "<=": np.less_equal, ">": np.greater, ">=": np.greater_equal}
    groups = [(sid, ts, cols) for sid, cgs in truth.items() for ts, cols in cgs]
    tps = np.nonzero(descs["phys_type"] == cabi.TSKV_PT_TIME)[0]
    assert len(tps) == len(groups)
    sel = None if sel is None else set(int(x) for x in sel)
    pages = nbytes = pruned = 0
    for k, (sid, ts, cols) in enumerate(groups):
        tp = int(tps[k])
        end = int(tps[k + 1]) if k + 1 < len(tps) else len(descs)
        assert int(descs[tp]["series_id"]) == sid and int(descs[tp]["num_values"]) == len(ts)
        if sel is not None and sid not in sel:
            continue
        q = [p for p in range(tp + 1, end) if int(descs[p]["column_id"]) in qcols]
        if not q:
            continue
        keep = not ranges or any(ts.min() <= hi and ts.max() >= lo for lo, hi in ranges)
        for col, pt, op, c in preds:
            if keep and col in cols:
                v, valid = cols[col]
                v = v[valid]
                keep = v.size > 0 and bool(ops[op](v.min(), c) or ops[op](v.max(), c))
        if keep:
            pages += len(q) + 1
            nbytes += sum(int(descs[p]["size"]) for p in q) + int(descs[tp]["size"])
        else:
            pruned += len(q)
    return pages, nbytes, pruned


def many_groups_arena(rng, groups, max_rows, fields=FIELDS, overlap_every=0, t0=1_000_000):
    """groups: {series id: column groups}. A series' groups follow each other in time, 1..max_rows rows each; with
    overlap_every = k, every k-th group starts inside the one before it. Returns (arena, descs, truth, file id of every
    column group: one chunk per group)."""
    b = datagen.ArenaBuilder()
    truth, files = {}, []
    for sid, n_cg in groups.items():
        t = t0
        for g in range(n_cg):
            n = int(rng.integers(1, max_rows + 1))
            if overlap_every and g % overlap_every == overlap_every - 1:
                t -= 500 * int(rng.integers(1, 40))
            ts = t + np.arange(n, dtype=np.int64) * 1000
            t = int(ts[-1]) + 1000
            fl, cols = [], {}
            for col, pt in fields:
                valid = rng.random(n) > 0.1
                if pt == cabi.TSKV_PT_F64:
                    v = np.cumsum(rng.integers(-3, 4, n)) + rng.random(n)
                elif pt == cabi.TSKV_PT_U64:
                    v = np.cumsum(rng.integers(0, 5, n)).astype(np.uint64)
                else:
                    v = np.cumsum(rng.integers(-9, 10, n)).astype(np.int64)
                fl.append((col, pt, v, valid))
                cols[col] = (v, valid)
            b.add_column_group(sid, ts, fl)
            truth.setdefault(sid, []).append((ts, cols))
            files.append(len(files) + 1)
    arena, descs = b.finish()
    return arena, descs, truth, files


def check_reads(engine, pages, arena, descs, truth, sel, kw, what, value_stats=True):
    """value_stats=False: a host-resident page set without caller-supplied statistics (no value-statistics pruning)."""
    q = make_query(FIELDS[:2], aggs=AGGS + ("first", "last"), series_ids=sel, **kw)
    assert_results_equal(engine.scan_aggregate(pages, q), orc.scan_aggregate(arena, descs, q, n_threads=8), what=what)
    c = engine.counters()
    got = (c["page_read_count"], c["page_read_bytes"], c["pruned_page_count"])
    exp = expected_reads(descs, truth, (1, 2), sel, kw.get("time_ranges", ()), kw.get("predicates", ()) if value_stats else ())
    assert got == exp, "%s: read / bytes / pruned %s, expected %s" % (what, got, exp)


def test_work_list_reads_exactly_the_selected_pages(engine):
    """The work list against the oracle and against reader counters restated from the arrays, with a selection list,
    without one, with time pruning and with value-statistics pruning plus the row filter, on two shapes: 2000 series of
    one column group each (one walk thread per series) and 6 series x 150 groups (8 walk threads per series). Column 3
    is never queried, so the counters must leave its pages out."""
    rng = np.random.default_rng(77)
    t0 = 1_000_000
    shapes = (("one group per series", {sid: 1 for sid in range(2000)}, 300, np.arange(0, 2000, 7, dtype=np.uint32)),
              ("many groups", {sid: 150 for sid in (2, 3, 5, 8, 13, 21)}, 80, np.array([3, 8, 21], dtype=np.uint32)))
    for shape, groups, max_rows, sel in shapes:
        arena, descs, truth, _ = many_groups_arena(rng, groups, max_rows)
        t_end = max(int(ts.max()) for cgs in truth.values() for ts, _ in cgs)
        w = (t_end - t0) // 40 + 1
        fbs, nb = bucket_spec(t0, t_end, w)
        pages = engine.upload_pages(arena, descs)
        for s in (sel, None):
            for kw in (dict(), dict(time_ranges=[(t0 + 40_000, t0 + 250_000), (t0 + 2_000_000, t0 + 3_000_000)]),
                       dict(predicates=[(1, cabi.TSKV_PT_I64, ">", 10)])):
                check_reads(engine, pages, arena, descs, truth, s, dict(width=w, first_bucket_start=fbs, n_buckets=nb,
                                                                       group_by_series=True, **kw),
                            "%s sel=%s %s" % (shape, s is not None, kw))
        pages.close()


def test_few_series_with_many_column_groups(engine):
    """3 series x 90 column groups: the work-list walk splits each series over 4 threads (at most 32 groups per
    thread). Results as the oracle's and reader counters as restated from the arrays, with time ranges, predicates
    (value-statistics pruning and the row filter), tombstones, FIRST / LAST, a host-resident page set and overlapping
    chunk files (every 7th group overlaps the one before it: merge groups between groups the walk reads)."""
    rng = np.random.default_rng(8)
    arena, descs, truth, files = many_groups_arena(rng, {4: 90, 9: 90, 11: 90}, 400)
    pages = engine.upload_pages(arena, descs)
    host = engine.upload_pages(arena, descs, host_resident=True)
    t0 = 1_000_000
    fbs, nb = bucket_spec(t0, t0 + 90 * 400 * 1000, 500_000)
    grid = dict(width=500_000, first_bucket_start=fbs, n_buckets=nb, group_by_series=True)
    preds = [(1, cabi.TSKV_PT_I64, ">", -20), (2, cabi.TSKV_PT_F64, "<=", 9.5)]
    for sel in (None, np.array([4, 11], dtype=np.uint32)):
        for kw in (dict(), dict(time_ranges=[(t0 + 3_000_000, t0 + 9_000_000)]), dict(predicates=preds),
                   dict(time_ranges=[(t0 + 1_000_000, t0 + 20_000_000)], predicates=preds[:1])):
            what = "many groups sel=%s %s" % (sel is not None, kw)
            check_reads(engine, pages, arena, descs, truth, sel, dict(grid, **kw), what)
            check_reads(engine, host, arena, descs, truth, sel, dict(grid, **kw), "host-resident " + what, value_stats=False)
            q = make_query(FIELDS[:2], aggs=AGGS + ("first", "last"), series_ids=sel, **grid, **kw)
            _, pts = orc.scan_aggregate(arena, descs, q, return_points=True)
            engine.scan_aggregate(pages, q)
            assert engine.counters()["points_decoded"] == pts
    host.close()
    tombs = random_tombstones(rng, descs, t0, t0 + 90 * 200 * 1000)
    pages.set_tombstones(tombs)
    for sel in (None, np.array([9], dtype=np.uint32)):
        q = make_query(FIELDS[:2], aggs=AGGS + ("first", "last"), series_ids=sel, time_ranges=[(t0 + 500_000, t0 + 30_000_000)], **grid)
        assert_results_equal(engine.scan_aggregate(pages, q), orc.scan_aggregate(arena, descs, q, tombstones=tombs),
                             what="tombstones sel=%s" % (sel is not None))
    pages.close()

    arena, descs, truth, files = many_groups_arena(rng, {4: 90, 9: 90, 11: 90}, 300, overlap_every=7)
    pages = engine.upload_pages(arena, descs)
    pages.set_chunk_files(files)
    for sel in (None, np.array([4, 11], dtype=np.uint32)):
        for kw in (dict(), dict(predicates=preds)):
            q = make_query(FIELDS[:2], aggs=AGGS + ("first", "last"), series_ids=sel, **grid, **kw)
            assert_results_equal(engine.scan_aggregate(pages, q), orc.scan_aggregate(arena, descs, q, chunk_files=files),
                                 what="overlapping chunks sel=%s %s" % (sel is not None, kw))
    pages.close()


def test_skewed_page_set_caps_the_walk_threads(engine):
    """One series of 1000 column groups among 3000 single-group series (12 000 field pages). The large series wants 32
    walk threads, but the walk may not launch more threads than there are field pages: 2000 selected series get 4
    threads each, all 3001 series 2 each. Results and reader counters as without the split."""
    rng = np.random.default_rng(31)
    groups = {0: 1000}
    groups.update({sid: 1 for sid in range(1, 3001)})
    arena, descs, truth, _ = many_groups_arena(rng, groups, 30)
    pages = engine.upload_pages(arena, descs)
    t0 = 1_000_000
    fbs, nb = bucket_spec(t0, t0 + 1000 * 30 * 1000, 2_000_000)
    sel = np.concatenate([[0], rng.choice(np.arange(1, 3001), 1999, replace=False)]).astype(np.uint32)
    sel.sort()
    for s in (sel, None):
        for kw in (dict(), dict(time_ranges=[(t0 + 15_000, t0 + 9_000_000)]), dict(predicates=[(1, cabi.TSKV_PT_I64, ">", 3)])):
            check_reads(engine, pages, arena, descs, truth, s, dict(width=2_000_000, first_bucket_start=fbs, n_buckets=nb, **kw),
                        "skewed sel=%s %s" % (s is not None, kw))
    pages.close()
