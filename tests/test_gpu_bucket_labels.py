"""Labelled time buckets (tskvgpu_scan_prepare_labels: GROUP BY date_part(unit, time) / EXTRACT(unit FROM time)).

1. Identity labels (labels[b] = b, n_buckets = n_edge) give the edge scan's result bit for bit (f64 SUM / MEAN within
   1e-12 relative) and the same counters, on RLE, jittered simple8b and raw (generic) time pages, narrow and wide
   simple8b values, a host-resident page set, time ranges, predicates, GROUP BY series and tag groups.
2. Cyclic labels over irregular and calendar edges (hour, minute, dow, month) on data spanning many periods, against the
   exact reference: i64 / u64 / f64 / bool columns, NULLs, time ranges, a predicate, tombstones and the overlap merge.
3. The labelled scan equals the host fold of the edge scan's COUNT / integer SUM / MIN / MAX over the same edges.
4. GROUP BY tags x labels and GROUP BY series x labels against the grouped reference.
5. Refusals, FIRST / LAST included. 6. A two-shard exchange and graph replay."""
import copy
import ctypes as C
import functools

import numpy as np
import pytest

from cnosdb_b200 import cabi
from cnosdb_b200.engine import PushedAggregate, QueryOption, TskvError, calendar_parts
from tests import exact_arenas as ea
from tests.helpers import ReferenceError, assert_matches_exact, make_query, random_arena
from tests.labels_reference import exact_aggregate_grouped_labels, exact_aggregate_labels
from tests.test_gpu_bucket_edges import assert_same_result, edge_query, paths_arena, random_edges, span
from tests.test_gpu_parity import random_tombstones

pytestmark = pytest.mark.gpu

ENVS = ("1", "3")  # TSKV_PARTS
FIELDS = ((1, cabi.TSKV_PT_I64), (2, cabi.TSKV_PT_F64), (3, cabi.TSKV_PT_U64))
PLAIN = ("count", "sum", "min", "max", "mean")
COUNTERS = ("points_decoded", "rows_in_range", "page_read_count", "pruned_page_count")
HOUR = 3600 * 10**9


def label_query(q, n_out):
    """q with its bucket grid replaced by n_out output buckets (the edges and labels come with the call)."""
    out = copy.copy(q)
    out.width, out.origin, out.first_bucket_start, out.n_buckets = 0, 0, 0, int(n_out)
    out._keep = None
    return out


def _scan(engine, pages, q, **kw):
    try:
        return engine.scan_aggregate(pages, q, **kw), None
    except TskvError as e:
        return None, e.status


def _counters(engine):
    c = engine.counters()
    return {k: c[k] for k in COUNTERS}


def check_vs_exact(engine, pages, truth, q, e, lab, what, extra=None, tombstones=None, files=None):
    """One labelled scan against the exact reference, status included."""
    extra = extra or {}
    try:
        if "group_ids" in extra:
            exp = exact_aggregate_grouped_labels(truth, q, extra["group_ids"], extra["n_groups"], e, lab,
                                                 tombstones=tombstones, files=files)
        else:
            exp = exact_aggregate_labels(truth, q, e, lab, tombstones=tombstones, files=files)
        err = None
    except ReferenceError as x:
        exp, err = None, x.status
    got, st = _scan(engine, pages, q, edges=e, labels=lab, group_ids=extra.get("group_ids"), n_groups=extra.get("n_groups"))
    if err is not None:
        assert st == err, "%s: status %s, the reference predicts %s" % (what, st, err)
        return None
    assert st is None, "%s: status %s" % (what, st)
    assert_matches_exact(got, exp, what=what)
    return got


# ---- 1. identity labels == the edge scan ----------------------------------------------------------------------------
def check_identity(engine, pages, q, e, what, **kw):
    qe, _ = edge_query(q, e)
    ref, st = _scan(engine, pages, qe, edges=e, **kw)
    ct = _counters(engine)
    got, sl = _scan(engine, pages, qe, edges=e, labels=np.arange(e.size - 1), **kw)
    assert sl == st, "%s: labelled status %s, edges %s" % (what, sl, st)
    if st is None:
        assert _counters(engine) == ct, "%s: counters %s vs %s" % (what, _counters(engine), ct)
        assert_same_result(got, ref, what)


def plain_columns(fields):
    """Every field with PLAIN aggregates (booleans: COUNT / MIN / MAX)."""
    return [PushedAggregate(c, pt, ("count", "min", "max") if pt == cabi.TSKV_PT_BOOL else PLAIN) for c, pt in fields]


@pytest.mark.parametrize("kind", ea.FL_KINDS)
def test_identity_labels_time_codecs(engine, kind, monkeypatch):
    """RLE, jittered simple8b and raw time pages; narrow and wide simple8b integers, Gorilla floats, booleans, NULLs."""
    arena, descs, truth = ea.first_last_arena(kind)
    rng = np.random.default_rng(13)
    lo, hi = span(truth)
    cols = plain_columns(ea.FL_FIELDS)
    ids = np.arange(ea.FL_SERIES, dtype=np.uint32)
    queries = [("plain", QueryOption(cols), {}),
               ("ranges", QueryOption(cols, time_ranges=[(lo + 15_000, lo + 95_000)]), {}),
               ("predicate", QueryOption(cols, predicates=[(4, cabi.TSKV_PT_I64, ">=", 0)]), {}),
               ("by_series", QueryOption(cols, group_by_series=True), {}),
               ("tags", QueryOption(cols), {"group_ids": (ids * 7 % 3).astype(np.uint32), "n_groups": 3})]
    dev = engine.upload_pages(arena, descs)
    host = engine.upload_pages(arena, descs, host_resident=True)
    for e in (random_edges(rng, lo, hi, 30, True), np.array([lo, hi + 1], dtype=np.int64)):
        for pname, pages in (("device", dev), ("host", host)):
            for qname, q, extra in queries:
                for parts in ENVS:
                    monkeypatch.setenv("TSKV_PARTS", parts)
                    check_identity(engine, pages, q, e, "%s %s %s %d parts=%s" % (kind, pname, qname, e.size, parts), **extra)
    dev.close()
    host.close()


@pytest.mark.parametrize("jitter", [0, 200])
def test_identity_labels_paths(engine, jitter, monkeypatch):
    """Predicates, pruning ranges, tombstones, a host-resident page set, GROUP BY series and tag groups."""
    arena, descs, truth, tombs = paths_arena(jitter)
    lo, hi = span(truth)
    e = random_edges(np.random.default_rng(21 + jitter), lo, hi, 60, True)
    gmap = (np.arange(80) * 7 % 9).astype(np.uint32)
    queries = [
        ("plain", make_query(FIELDS, PLAIN), {}),
        ("ranges", make_query(FIELDS, PLAIN, time_ranges=[(lo + 50_000, lo + 333_333)]), {}),
        ("predicate", make_query(FIELDS, PLAIN, predicates=[(1, cabi.TSKV_PT_I64, ">", -20)]), {}),
        ("by_series", make_query(FIELDS, PLAIN, group_by_series=True), {}),
        ("tags", make_query(FIELDS, PLAIN), {"group_ids": gmap, "n_groups": 9}),
    ]
    dev = engine.upload_pages(arena, descs)
    host = engine.upload_pages(arena, descs, host_resident=True)
    tomb = engine.upload_pages(arena, descs)
    tomb.set_tombstones(tombs)
    for pname, pages in (("device", dev), ("host", host), ("tombstones", tomb)):
        for qname, q, extra in queries:
            for parts in ENVS:
                monkeypatch.setenv("TSKV_PARTS", parts)
                check_identity(engine, pages, q, e, "%s %s parts=%s" % (pname, qname, parts), **extra)
    for p in (dev, host, tomb):
        p.close()


# ---- 2. cyclic labels against the exact reference -------------------------------------------------------------------
T_PRE = -36 * HOUR  # 1969-12-30T12:00


@functools.lru_cache(maxsize=None)
def cyclic_arena(jitter):
    """40 series, one row every 37 s for ~3 days from 36 hours before 1970 (many hours and minutes per page), 10 %
    NULLs, i64 / f64 / u64 fields."""
    rng = np.random.default_rng(61 + jitter)
    return random_arena(rng, n_series=40, n_points=7000, fields=FIELDS, null_frac=0.1, t0=T_PRE, step=37 * 10**9,
                        jitter=jitter)


@functools.lru_cache(maxsize=None)
def calendar_arena(jitter):
    """40 series, one row every 23 hours from February 1968 for ~4.7 years (rows before and after 1970)."""
    rng = np.random.default_rng(81 + jitter)
    t0 = int(np.datetime64("1968-02-10T05:00:00", "ns").astype(np.int64))
    return random_arena(rng, n_series=40, n_points=1800, fields=FIELDS, null_frac=0.1, t0=t0, step=23 * HOUR,
                        jitter=jitter)


@pytest.mark.parametrize("jitter", [0, 5 * 10**9])
@pytest.mark.parametrize("unit", ["hour", "minute"])
def test_cyclic_hour_minute(engine, unit, jitter, monkeypatch):
    arena, descs, truth = cyclic_arena(jitter)
    pages = engine.upload_pages(arena, descs)
    lo, hi = span(truth)
    e, lab, values = calendar_parts(unit, lo, hi)
    assert e.size - 1 > 2 * values.size  # every output bucket folds several periods
    gmap = (np.arange(40) % 4).astype(np.uint32)
    for extra, kw in (({}, {}), ({}, {"group_by_series": True}), ({"group_ids": gmap, "n_groups": 4}, {}),
                      ({}, {"time_ranges": [(0, hi - HOUR)], "predicates": [(1, cabi.TSKV_PT_I64, "<=", 10)]})):
        q = label_query(make_query(FIELDS, PLAIN, **kw), values.size)
        for parts in ENVS:
            monkeypatch.setenv("TSKV_PARTS", parts)
            check_vs_exact(engine, pages, truth, q, e, lab, "%s jitter=%d %s %s parts=%s" % (unit, jitter, kw, bool(extra),
                                                                                             parts), extra)
    pages.close()


@pytest.mark.parametrize("jitter", [0, 3 * 10**12])
@pytest.mark.parametrize("unit", ["dow", "month", "day", "week", "year"])
def test_cyclic_calendar(engine, unit, jitter, monkeypatch):
    arena, descs, truth = calendar_arena(jitter)
    pages = engine.upload_pages(arena, descs)
    e, lab, values = calendar_parts(unit, *span(truth))
    assert e[0] < 0 < e[-1]
    gmap = (np.arange(40) % 4).astype(np.uint32)
    for extra, kw in (({}, {}), ({}, {"group_by_series": True}), ({"group_ids": gmap, "n_groups": 4}, {}),
                      ({}, {"time_ranges": [(0, int(e[-1]))]})):
        q = label_query(make_query(FIELDS, PLAIN, **kw), values.size)
        for parts in ENVS:
            monkeypatch.setenv("TSKV_PARTS", parts)
            check_vs_exact(engine, pages, truth, q, e, lab, "%s jitter=%d %s %s parts=%s" % (unit, jitter, kw, bool(extra),
                                                                                             parts), extra)
    pages.close()


def test_cyclic_irregular_edges(engine, monkeypatch):
    """Random edges (some narrower than the time step: empty edge buckets), labels b % k, output buckets no edge bucket
    maps to; tombstones."""
    arena, descs, truth, tombs = paths_arena()
    rng = np.random.default_rng(93)
    lo, hi = span(truth)
    pages = engine.upload_pages(arena, descs)
    tp = engine.upload_pages(arena, descs)
    tp.set_tombstones(tombs)
    for n, k, n_out in ((40, 7, 7), (300, 5, 9), (3000, 60, 64)):
        e = random_edges(rng, lo, hi, n, True)
        lab = (np.arange(e.size - 1) % k).astype(np.uint32)
        for extra, kw in (({}, {}), ({}, {"group_by_series": True}),
                          ({}, {"predicates": [(1, cabi.TSKV_PT_I64, "<=", 10)], "time_ranges": [(lo + 5000, hi - 5000)]})):
            q = label_query(make_query(FIELDS, PLAIN, **kw), n_out)
            for parts in ENVS:
                monkeypatch.setenv("TSKV_PARTS", parts)
                what = "n=%d k=%d %s parts=%s" % (n, k, kw, parts)
                check_vs_exact(engine, pages, truth, q, e, lab, what, extra)
                check_vs_exact(engine, tp, truth, q, e, lab, what + " tombstones", extra, tombstones=tombs)
    pages.close()
    tp.close()


def _cyclic(q, rng, k=3):
    """q's grid span cut at random points, labelled b % k -> (query, edges, labels)."""
    lo = q.first_bucket_start
    hi = lo + q.n_buckets * q.width - 1
    e = random_edges(rng, lo, hi, max(2, q.n_buckets * 2 // 3), True)
    return label_query(q, k), e, (np.arange(e.size - 1) % k).astype(np.uint32)


def _plain(q):
    """q with its FIRST / LAST dropped (booleans keep COUNT / MIN / MAX)."""
    out = copy.copy(q)
    out.columns = [PushedAggregate(c.column_id, c.phys_type, c.agg_mask & ~(cabi.TSKV_AGG_FIRST | cabi.TSKV_AGG_LAST))
                   for c in q.columns]
    out._keep = None
    return out


@pytest.mark.parametrize("kind", ea.FL_KINDS)
def test_bool_and_null_pages(engine, kind):
    """i64 / u64 / f64 / bool columns with NULL runs and raw value pages, the row filter and tag groups."""
    arena, descs, truth = ea.first_last_arena(kind)
    pages = engine.upload_pages(arena, descs)
    rng = np.random.default_rng(15)
    for name, q, extra in ea.first_last_queries(truth):
        if q.width <= 0:
            continue
        qe, e, lab = _cyclic(_plain(q), rng)
        check_vs_exact(engine, pages, truth, qe, e, lab, "%s %s" % (kind, name), extra)
    pages.close()


@pytest.mark.parametrize("step,kind", ea.TB_CASES)
def test_tombstones(engine, step, kind):
    arena, descs, truth = ea.tombstone_arena(step, kind)
    tombs = ea.tombstone_list(truth, step)
    pages = engine.upload_pages(arena, descs)
    pages.set_tombstones(tombs)
    rng = np.random.default_rng(16)
    for name, q, extra in ea.tombstone_queries(truth, step):
        if q.width <= 0 or "slide" in extra:
            continue
        qe, e, lab = _cyclic(_plain(q), rng)
        check_vs_exact(engine, pages, truth, qe, e, lab, "%d %s %s" % (step, kind, name), extra, tombstones=tombs)
    pages.close()


@pytest.mark.parametrize("tombstoned", [False, True])
def test_overlap_merge(engine, tombstoned):
    arena, descs, truth, files = ea.merge_arena()
    tombs = ea.merge_tombstones(truth) if tombstoned else None
    pages = engine.upload_pages(arena, descs)
    pages.set_chunk_files(files)
    if tombstoned:
        pages.set_tombstones(tombs)
    rng = np.random.default_rng(17)
    for name, q, extra in ea.merge_queries(truth):
        if q.width <= 0:
            continue
        qe, e, lab = _cyclic(_plain(q), rng)
        check_vs_exact(engine, pages, truth, qe, e, lab, "merge %s tombstones=%s" % (name, tombstoned), extra,
                       tombstones=tombs, files=files)
    pages.close()


# ---- 3. the host fold of the edge scan -----------------------------------------------------------------------------
@pytest.mark.parametrize("jitter", [0, 5 * 10**9])
def test_labels_equal_folded_edge_scan(engine, jitter, monkeypatch):
    arena, descs, truth = cyclic_arena(jitter)
    pages = engine.upload_pages(arena, descs)
    lo, hi = span(truth)
    aggs = ("count", "sum", "min", "max")
    for unit in ("minute", "hour"):
        e, lab, values = calendar_parts(unit, lo, hi)
        for kw in ({}, {"group_by_series": True}):
            q = make_query(FIELDS, aggs, **kw)
            for parts in ENVS:
                monkeypatch.setenv("TSKV_PARTS", parts)
                qe, _ = edge_query(q, e)
                fine = engine.scan_aggregate(pages, qe, edges=e)
                got = engine.scan_aggregate(pages, label_query(q, values.size), edges=e, labels=lab)
                for col, agg in got.names:
                    what = "%s %s parts=%s col %s %s" % (unit, kw, parts, col, agg)
                    v, ok = fine.column(col, agg)
                    g, gok = got.column(col, agg)
                    for r in range(v.shape[0]):
                        exp_ok = np.bincount(lab, weights=ok[r], minlength=values.size) > 0
                        assert (gok[r] == exp_ok).all(), what
                        if agg == "sum" and got.phys[col] == cabi.TSKV_PT_F64:
                            continue  # (float sums: the order of the additions differs)
                        exp = np.zeros(values.size, dtype=v.dtype)
                        for j in range(values.size):
                            m = ok[r] & (lab == j)
                            if not m.any():
                                continue
                            if agg in ("count", "sum"):
                                with np.errstate(over="ignore"):
                                    exp[j] = v[r][m].sum(dtype=v.dtype)
                            else:
                                exp[j] = v[r][m].min() if agg == "min" else v[r][m].max()
                        assert (g[r][gok[r]] == exp[gok[r]]).all(), what
    pages.close()


# ---- 5. refusals ----------------------------------------------------------------------------------------------------
def _arg(a, dtype):
    return None if a is None else np.ascontiguousarray(a, dtype=dtype)


def _layout_status(engine, pages, q, e, n_edge, lab, gids=None, n_groups=0):
    L = cabi.OutputLayout()
    qc = q.to_c()
    ep, lp, gp = _arg(e, np.int64), _arg(lab, np.uint32), _arg(gids, np.uint32)
    return engine.lib.tskvgpu_query_output_layout_labels(
        pages.handle, C.byref(qc), None if ep is None else ep.ctypes.data, n_edge, None if lp is None else lp.ctypes.data,
        None if gp is None else gp.ctypes.data, n_groups, C.byref(L))


def _prepare_status(engine, pages, q, e, n_edge, lab, gids=None, n_groups=0):
    qc = q.to_c()
    ep, lp, gp = _arg(e, np.int64), _arg(lab, np.uint32), _arg(gids, np.uint32)
    h = C.c_void_p()
    st = engine.lib.tskvgpu_scan_prepare_labels(
        engine.ctx, pages.handle, C.byref(qc), None if ep is None else ep.ctypes.data, n_edge,
        None if lp is None else lp.ctypes.data, None if gp is None else gp.ctypes.data, n_groups, C.byref(h))
    if h.value:
        engine.lib.tskvgpu_scan_destroy(engine.ctx, h)
    return st


def _aggregate_status(engine, pages, q, e, n_edge, lab):
    qc = q.to_c()
    ep, lp = _arg(e, np.int64), _arg(lab, np.uint32)
    values = np.zeros(1 << 16, dtype=np.uint64)
    bitmaps = np.zeros(1 << 16, dtype=np.uint8)
    return engine.lib.tskvgpu_scan_aggregate_labels(
        engine.ctx, pages.handle, C.byref(qc), None if ep is None else ep.ctypes.data, n_edge,
        None if lp is None else lp.ctypes.data, None, 0, values.ctypes.data, bitmaps.ctypes.data)


def test_refusals(engine):
    arena, descs, truth = random_arena(np.random.default_rng(3), n_series=129, n_points=50, fields=FIELDS)
    pages = engine.upload_pages(arena, descs)
    good = np.array([0, 1_020_000, 1_040_000, 1_060_000], dtype=np.int64)
    lab = np.array([0, 1, 0], dtype=np.uint32)
    base = label_query(make_query(FIELDS, PLAIN), 2)
    INV, UNS = cabi.TSKV_ERR_INVALID_ARG, cabi.TSKV_ERR_UNSUPPORTED

    def variant(**kw):
        q = copy.copy(base)
        q._keep = None
        for k, v in kw.items():
            setattr(q, k, v)
        return q
    cases = [
        ("labels NULL", base, good, 3, None, None, 0),
        ("label >= n_buckets", variant(n_buckets=1), good, 3, lab, None, 0),
        ("label far out", base, good, 3, np.array([0, 2**32 - 1, 0]), None, 0),
        ("n_buckets 0", variant(n_buckets=0), good, 3, np.zeros(3), None, 0),
        ("edges NULL", base, None, 3, lab, None, 0),
        ("n_edge 0", base, good, 0, lab, None, 0),
        ("not increasing", base, np.array([0, 5, 5, 1_060_000]), 3, lab, None, 0),
        ("decreasing", base, np.array([0, 1_060_000, 5, 1_070_000]), 3, lab, None, 0),
        ("span 2^63", base, np.array([-2**63, 0, 1]), 2, lab[:2], None, 0),
        ("width", variant(width=20_000), good, 3, lab, None, 0),
        ("origin", variant(origin=1), good, 3, lab, None, 0),
        ("first_bucket_start", variant(first_bucket_start=1), good, 3, lab, None, 0),
        ("group id >= n_groups", base, good, 3, lab, np.full(129, 3, np.uint32), 3),
        ("n_groups 0", base, good, 3, lab, np.zeros(129, np.uint32), 0),
        ("group map with group_by_series", variant(group_by_series=True), good, 3, lab, np.zeros(129, np.uint32), 1),
        ("cells > TSKV_MAX_GROUPED_CELLS", base, good, 3, lab, np.zeros(129, np.uint32), 2**31),
    ]
    for what, q, e, n_edge, lb, gids, ng in cases:
        assert _layout_status(engine, pages, q, e, n_edge, lb, gids, ng) == INV, what
        assert _prepare_status(engine, pages, q, e, n_edge, lb, gids, ng) == INV, what
    for what, q, e, n_edge, lb, gids, ng in cases[:12]:
        assert _aggregate_status(engine, pages, q, e, n_edge, lb) == INV, what
    # the largest span and a label table that leaves output buckets unused are accepted
    assert _layout_status(engine, pages, base, np.array([-2**63, -1]), 1, np.array([1])) == cabi.TSKV_OK
    assert _layout_status(engine, pages, variant(n_buckets=2**20), good, 3, lab) == cabi.TSKV_OK
    # FIRST / LAST: refused, whatever the key budget (one series, GROUP BY series)
    for aggs in (("count", "first"), ("last",), ("count", "sum", "first", "last")):
        for kw in ({}, {"group_by_series": True}, {"series_ids": np.array([0], np.uint32)}):
            q = label_query(make_query(FIELDS, aggs, **kw), 2)
            assert _layout_status(engine, pages, q, good, 3, lab) == UNS, (aggs, kw)
            assert _prepare_status(engine, pages, q, good, 3, lab) == UNS, (aggs, kw)
            assert _aggregate_status(engine, pages, q, good, 3, lab) == UNS, (aggs, kw)
            with pytest.raises(TskvError) as err:
                engine.prepare(pages, q, edges=good, labels=lab)
            assert err.value.status == UNS
    # the Python layer: labels need edges, one label per edge bucket, no sliding windows
    with pytest.raises(ValueError):
        engine.scan_aggregate(pages, base, labels=lab)
    with pytest.raises(ValueError):
        engine.scan_aggregate(pages, base, edges=good, labels=lab[:2])
    with pytest.raises(ValueError):
        engine.prepare(pages, base, slide=10, edges=good, labels=lab)
    pages.close()


@pytest.mark.parametrize("jitter", [0, 300])
def test_row_outside_the_edges(engine, jitter):
    """A selected row before edges[0] or at / after edges[n_edge]: TSKV_ERR_BUCKET_RANGE, as in the edge scan."""
    arena, descs, truth = random_arena(np.random.default_rng(4), n_series=40, n_points=300, fields=FIELDS, jitter=jitter)
    pages = engine.upload_pages(arena, descs)
    lo, hi = span(truth)
    for e in (np.array([lo + 1, lo + 9000, hi + 1]), np.array([lo, lo + 1000, lo + 50_000, hi])):
        lab = (np.arange(e.size - 1) % 2).astype(np.uint32)
        q = label_query(make_query(FIELDS, PLAIN), 2)
        with pytest.raises(ReferenceError):
            exact_aggregate_labels(truth, q, e, lab)
        with pytest.raises(TskvError) as err:
            engine.scan_aggregate(pages, q, edges=e, labels=lab)
        assert err.value.status == cabi.TSKV_ERR_BUCKET_RANGE
        assert 0 <= err.value.page < len(descs)
        qr = copy.copy(q)
        qr.time_ranges, qr._keep = [(int(e[0]), int(e[-1]) - 1)], None
        check_vs_exact(engine, pages, truth, qr, e, lab, "clipped %s" % (e,))
    pages.close()


# ---- 6. two-shard exchange, graph replay ----------------------------------------------------------------------------
def test_two_shard_exchange(engine):
    """Two series shards scanned separately with the same edges and labels, their exchange regions concatenated like an
    all-gather and merged: every rank's result equals the exact reference over both shards."""
    import torch
    from cnosdb_b200.parallel import device_tensor
    arena, descs, truth = cyclic_arena(5 * 10**9)
    e, lab, values = calendar_parts("hour", *span(truth))
    ids = np.arange(40, dtype=np.uint32)
    dev = torch.device("cuda", engine.device)
    for gbs in (False, True):
        q = label_query(make_query(FIELDS, PLAIN, series_ids=ids, group_by_series=gbs, multi_rank=True), values.size)
        exp = exact_aggregate_labels(truth, q, e, lab)
        scans, regions, keep = [], [], []
        for shard in (ids[ids % 2 == 0], ids[ids % 2 == 1]):
            pages = engine.upload_pages(arena, descs[np.isin(descs["series_id"], shard)])
            s = engine.prepare(pages, q, edges=e, labels=lab)
            s.run()
            ptr, words = s.exchange_view()
            regions.append(device_tensor(ptr, words, torch.int64, dev).clone())
            scans.append(s)
            keep.append(pages)
        gathered = torch.cat(regions)
        torch.cuda.synchronize()
        for s in scans:
            s.merge_gathered(gathered.data_ptr(), 2)
            assert_matches_exact(s.finalize(), exp, what="2-shard exchange gbs=%s" % gbs, int_mean=False)
            s.close()
        for p in keep:
            p.close()


def test_graph_replay(engine):
    arena, descs, truth = cyclic_arena(0)
    pages = engine.upload_pages(arena, descs)
    for unit in ("hour", "minute"):
        e, lab, values = calendar_parts(unit, *span(truth))
        q = label_query(make_query(FIELDS, PLAIN), values.size)
        once = engine.scan_aggregate(pages, q, edges=e, labels=lab)
        assert_matches_exact(once, exact_aggregate_labels(truth, q, e, lab), what="graph replay %s once" % unit)
        s = engine.prepare(pages, q, edges=e, labels=lab)
        for _ in range(4):  # the second enqueue captures the pass as a CUDA graph, the later ones replay it
            s.enqueue()
            s.sync()
            assert_same_result(s.finalize(), once, "graph replay %s" % unit)
        s.close()
    pages.close()
