"""Explicit time-bucket edges (tskvgpu_scan_prepare_edges: GROUP BY date_trunc(unit, time) and other irregular grids).

1. The tumbling grid handed in as edges gives the tumbling scan's result bit for bit (f64 SUM / MEAN within 1e-12
   relative: the order of the sums differs) and the same counters, on the bucket-geometry arenas (RLE, simple8b and
   generic timestamps) and with predicates, tombstones, a host-resident page set, GROUP BY series and tag groups.
2. Irregular edges (calendar months / years / weeks with rows before 1970, random edges with empty cells, one bucket over
   everything) against the exact reference, with FIRST / LAST ties, tombstones, the row filter, the overlap merge, tag
   groups and GROUP BY series.
3. Edges on every m-th line of a uniform grid == m tumbling buckets folded on the host (COUNT / SUM / MIN / MAX).
4. Refusals, 5. a two-shard exchange with FIRST / LAST, 6. graph replay."""
import copy
import ctypes as C
import functools

import numpy as np
import pytest

from cnosdb_b200 import cabi
from cnosdb_b200.engine import TskvError, calendar_edges
from tests import exact_arenas as ea
from tests.edges_reference import exact_aggregate_edges, exact_aggregate_grouped_edges
from tests.helpers import (ALL_AGGS, GEOMETRY_CASES, I64_MAX, I64_MIN, ReferenceError, assert_matches_exact,
                           bucket_spec, exact_aggregate, geometry_arena, geometry_queries, geometry_ranges, make_query,
                           random_arena)
from tests.test_gpu_parity import random_tombstones

pytestmark = pytest.mark.gpu

ENVS = ("1", "3")  # TSKV_PARTS
FIELDS = ((1, cabi.TSKV_PT_I64), (2, cabi.TSKV_PT_F64), (3, cabi.TSKV_PT_U64))
PLAIN = ("count", "sum", "min", "max", "mean")
DAY = 86400 * 10**9
COUNTERS = ("points_decoded", "rows_in_range", "page_read_count")


def edge_query(q, edges):
    """q with its bucket grid replaced by the explicit edges -> (query, int64 edges)."""
    e = np.asarray(edges, dtype=np.int64)
    out = copy.copy(q)
    out.width, out.origin, out.first_bucket_start, out.n_buckets = 0, 0, 0, int(e.size - 1)
    out._keep = None
    return out, e


def span(truth):
    """(min, max) time of the arena's rows."""
    ts = np.concatenate([t for cgs in truth.values() for t, _ in cgs])
    return int(ts.min()), int(ts.max())


def grid_edges(q):
    return np.array([q.first_bucket_start + j * q.width for j in range(q.n_buckets + 1)], dtype=np.int64)


def floor_grid(truth, q):
    """Does every row of the arena lie in the floor regime of q's grid (dividend t - origin % w + w >= 0, no wrap), and
    does the grid end inside the int64 range? Then the grid's edges put every row where the tumbling scan does."""
    if q.width <= 0:
        return False
    o = abs(q.origin) % q.width * (1 if q.origin >= 0 else -1)  # Rust's truncating %
    ts = [t for cgs in truth.values() for t, _ in cgs if len(t)]
    lo, hi = min(int(np.min(t)) for t in ts), max(int(np.max(t)) for t in ts)
    return (lo - o + q.width >= 0 and hi - o + q.width <= I64_MAX and
            q.first_bucket_start + q.n_buckets * q.width <= I64_MAX)


def _scan(engine, pages, q, **kw):
    try:
        return engine.scan_aggregate(pages, q, **kw), None
    except TskvError as e:
        return None, e.status


def _counters(engine):
    c = engine.counters()
    return {k: c[k] for k in COUNTERS}


def assert_same_result(got, exp, what, first_last=True):
    """GPU result vs GPU result: bit for bit, f64 SUM / MEAN within 1e-12 relative (NaN / inf equal)."""
    assert got.names == exp.names
    for j, (col, agg) in enumerate(got.names):
        if agg in ("first", "last") and not first_last:
            continue
        assert (got.validity[j] == exp.validity[j]).all(), "%s col %s %s: validity differs" % (what, col, agg)
        ok = got.validity[j]
        if agg in ("sum", "mean") and got.phys[col] == cabi.TSKV_PT_F64:
            g, e = got.values[j][ok].view(np.float64), exp.values[j][ok].view(np.float64)
            with np.errstate(invalid="ignore"):
                close = np.where(np.isnan(e), np.isnan(g), np.where(np.isinf(e), g == e,
                                                                   np.abs(g - e) <= 1e-12 * np.maximum(np.abs(e), 1e-300)))
            bad = np.nonzero(~close)[0]
            assert bad.size == 0, "%s col %s %s differs at %s: %s vs %s" % (what, col, agg, bad[:5], g[bad[:5]], e[bad[:5]])
        else:
            bad = np.nonzero(got.values[j][ok] != exp.values[j][ok])[0]
            assert bad.size == 0, "%s col %s %s differs at %s" % (what, col, agg, bad[:5])


def exact_edges(truth, q, e, extra=None, tombstones=None, files=None):
    extra = extra or {}
    if "group_ids" in extra:
        return exact_aggregate_grouped_edges(truth, q, extra["group_ids"], extra["n_groups"], e, tombstones=tombstones,
                                             files=files)
    return exact_aggregate_edges(truth, q, e, tombstones=tombstones, files=files)


def check_vs_exact(engine, pages, truth, q, e, what, extra=None, tombstones=None, files=None):
    """One edge scan against the exact reference, status included."""
    extra = extra or {}
    try:
        exp, err = exact_edges(truth, q, e, extra, tombstones, files), None
    except ReferenceError as x:
        exp, err = None, x.status
    got, st = _scan(engine, pages, q, edges=e, group_ids=extra.get("group_ids"), n_groups=extra.get("n_groups"))
    if err is not None:
        assert st == err, "%s: status %s, the reference predicts %s" % (what, st, err)
        return None
    assert st is None, "%s: status %s" % (what, st)
    assert_matches_exact(got, exp, what=what)
    return got


def check_same_as_tumbling(engine, pages, q, what, first_last=True, **kw):
    """The tumbling scan of q and the edge scan of q's own grid: equal results and counters (or the same refusal; a
    FIRST / LAST refusal of the tumbling scan's 2 * width budget may pass with the edges' longest-bucket budget)."""
    tum, st = _scan(engine, pages, q, **kw)
    ct = _counters(engine)
    qe, e = edge_query(q, grid_edges(q))
    got, se = _scan(engine, pages, qe, edges=e, **kw)
    if st is not None:
        if st != cabi.TSKV_ERR_UNSUPPORTED:
            assert se == st, "%s: edge scan status %s, tumbling %s" % (what, se, st)
        return None
    assert se is None, "%s: edge scan status %s" % (what, se)
    assert _counters(engine) == ct, "%s: counters %s vs %s" % (what, _counters(engine), ct)
    assert_same_result(got, tum, what, first_last)
    return got


# ---- 1. the tumbling grid as edges -------------------------------------------------------------------------------------
FLOOR_CASES = [c for c in GEOMETRY_CASES if c[4] > -2**61 and c[4] < 2**61 and c[2] < 2**61]


@pytest.mark.parametrize("case", FLOOR_CASES, ids=[c[0] for c in FLOOR_CASES])
def test_uniform_grid_equals_tumbling_geometry(engine, case, monkeypatch):
    name, step, w, origin, t0, n, kinds = case
    arena, descs, truth = geometry_arena(len(name), t0, step, n)
    pages = engine.upload_pages(arena, descs)
    ran = 0
    for kind in kinds:
        ranges = geometry_ranges(kind, t0, step, n, w, origin)
        for qname, q in geometry_queries(case, ranges, truth):
            if not floor_grid(truth, q) or q.n_buckets > 1 << 16:
                continue
            for parts in ENVS:
                monkeypatch.setenv("TSKV_PARTS", parts)
                check_same_as_tumbling(engine, pages, q, "%s %s %s parts=%s" % (name, kind, qname, parts),
                                       first_last=bool(step))
                ran += 1
    pages.close()
    if ran == 0:
        pytest.skip("no query of this case has a floor-regime grid")


@functools.lru_cache(maxsize=None)
def paths_arena(jitter=200):
    """80 series of 600 rows 1000 ns apart (jitter 0: RLE time pages, else simple8b), 10 % NULLs, some series in two
    column groups, a few raw-encoded value pages; and a tombstone list over them."""
    rng = np.random.default_rng(71 + jitter)
    arena, descs, truth = random_arena(rng, n_series=80, n_points=600, fields=FIELDS, null_frac=0.1, jitter=jitter,
                                       multi_cg=True, raw_frac=0.05)
    return arena, descs, truth, random_tombstones(np.random.default_rng(72), descs, *span(truth))


@pytest.mark.parametrize("jitter", [0, 200])
def test_uniform_grid_equals_tumbling_paths(engine, jitter, monkeypatch):
    """Predicates, tombstones, a host-resident page set, GROUP BY series and tag groups."""
    arena, descs, truth, tombs = paths_arena(jitter)
    lo, hi = span(truth)
    fbs, nb = bucket_spec(lo, hi, 20_000)
    grid = dict(width=20_000, first_bucket_start=fbs, n_buckets=nb)
    gmap = (np.arange(80) * 7 % 9).astype(np.uint32)
    queries = [
        ("bucket", make_query(FIELDS, PLAIN, **grid), {}),
        ("bucket+sel", make_query(FIELDS, ALL_AGGS, **grid), {}),
        ("ranges", make_query(FIELDS, ALL_AGGS, time_ranges=[(lo + 50_000, lo + 333_333)], **grid), {}),
        ("predicate", make_query(FIELDS, PLAIN, predicates=[(1, cabi.TSKV_PT_I64, ">", -20)], **grid), {}),
        ("predicate+sel", make_query(FIELDS, ALL_AGGS, predicates=[(2, cabi.TSKV_PT_F64, "<", 3.0)], **grid), {}),
        ("by_series", make_query(FIELDS, ALL_AGGS, group_by_series=True, **grid), {}),
        ("tags", make_query(FIELDS, PLAIN, **grid), {"group_ids": gmap, "n_groups": 9}),
        ("tags+sel", make_query(FIELDS, ALL_AGGS, **grid), {"group_ids": gmap, "n_groups": 9}),
    ]
    dev = engine.upload_pages(arena, descs)
    host = engine.upload_pages(arena, descs, host_resident=True)
    tomb = engine.upload_pages(arena, descs)
    tomb.set_tombstones(tombs)
    for pname, pages in (("device", dev), ("host", host), ("tombstones", tomb)):
        for qname, q, extra in queries:
            for parts in ENVS:
                monkeypatch.setenv("TSKV_PARTS", parts)
                check_same_as_tumbling(engine, pages, q, "%s %s parts=%s" % (pname, qname, parts), **extra)
    for p in (dev, host, tomb):
        p.close()


# ---- 2. irregular edges against the exact reference ----------------------------------------------------------------
T_1968 = int(np.datetime64("1968-02-10T05:00:00", "ns").astype(np.int64))


@functools.lru_cache(maxsize=None)
def calendar_arena(jitter):
    """40 series, one row every 23 hours from February 1968 for ~4.7 years (rows before and after 1970)."""
    rng = np.random.default_rng(81 + jitter)
    return random_arena(rng, n_series=40, n_points=1800, fields=FIELDS, null_frac=0.1, t0=T_1968, step=23 * 3600 * 10**9,
                        jitter=jitter)


@pytest.mark.parametrize("jitter", [0, 3_000_000_000_000])
@pytest.mark.parametrize("unit", ["month", "quarter", "year", "week"])
def test_calendar_units(engine, unit, jitter, monkeypatch):
    arena, descs, truth = calendar_arena(jitter)
    pages = engine.upload_pages(arena, descs)
    e = calendar_edges(unit, *span(truth))
    assert e[0] < 0 < e[-1]
    gmap = (np.arange(40) % 4).astype(np.uint32)
    for aggs in (PLAIN, ALL_AGGS):
        for extra, kw in (({}, {}), ({}, {"group_by_series": True}), ({"group_ids": gmap, "n_groups": 4}, {}),
                          ({}, {"time_ranges": [(0, int(e[-1]))]})):
            q, _ = edge_query(make_query(FIELDS, aggs, **kw), e)
            for parts in ENVS:
                monkeypatch.setenv("TSKV_PARTS", parts)
                check_vs_exact(engine, pages, truth, q, e, "%s jitter=%d %s %s %s parts=%s" % (unit, jitter, aggs, kw,
                                                                                               bool(extra), parts), extra)
    pages.close()


def random_edges(rng, lo, hi, n, narrow):
    """n + 1 increasing edges over [lo, hi + 1]: random cut points, some of them 1 apart (buckets narrower than the
    time step: empty cells)."""
    cuts = rng.integers(lo + 1, hi + 1, n - 1)
    if narrow:
        cuts = np.concatenate([cuts, cuts[: n // 4] + 1, cuts[: n // 8] + 2])
    return np.unique(np.concatenate([[lo], cuts, [hi + 1]])).astype(np.int64)


def test_random_edges(engine, monkeypatch):
    arena, descs, truth, tombs = paths_arena()
    rng = np.random.default_rng(91)
    lo, hi = span(truth)
    tables = [random_edges(rng, lo, hi, 40, False), random_edges(rng, lo, hi, 200, True),
              random_edges(rng, lo, hi, 3000, True),
              np.array([lo - 2**61, lo + 123_457, lo + 2**61], dtype=np.int64),  # (FIRST / LAST across series: refused)
              np.array([lo, hi + 1], dtype=np.int64)]  # (one bucket spanning everything)
    gmap = (np.arange(80) % 5).astype(np.uint32)
    pages = engine.upload_pages(arena, descs)
    tp = engine.upload_pages(arena, descs)
    tp.set_tombstones(tombs)
    for k, e in enumerate(tables):
        for aggs in (PLAIN, ALL_AGGS):
            for extra, kw in (({}, {}), ({}, {"group_by_series": True}), ({"group_ids": gmap, "n_groups": 5}, {}),
                              ({}, {"predicates": [(1, cabi.TSKV_PT_I64, "<=", 10)], "time_ranges": [(lo + 5000, hi - 5000)]})):
                q, _ = edge_query(make_query(FIELDS, aggs, **kw), e)
                for parts in ENVS:
                    monkeypatch.setenv("TSKV_PARTS", parts)
                    what = "table %d %s %s %s parts=%s" % (k, aggs, kw, bool(extra), parts)
                    check_vs_exact(engine, pages, truth, q, e, what, extra)
                    check_vs_exact(engine, tp, truth, q, e, what + " tombstones", extra, tombstones=tombs)
    pages.close()
    tp.close()


def _irregular(q, rng):
    """q's grid span cut at random points (some buckets narrower than the step)."""
    lo = q.first_bucket_start
    hi = lo + q.n_buckets * q.width - 1
    return edge_query(q, random_edges(rng, lo, hi, max(2, q.n_buckets * 2 // 3), True))


@pytest.mark.parametrize("kind", ea.FL_KINDS)
def test_first_last_runs_and_ties(engine, kind, monkeypatch):
    """The FIRST / LAST arenas: runs whose first / last row is NULL, ties across series at one time."""
    arena, descs, truth = ea.first_last_arena(kind)
    pages = engine.upload_pages(arena, descs)
    rng = np.random.default_rng(5)
    for name, q, extra in ea.first_last_queries(truth):
        if q.width <= 0 or "slide" in extra:
            continue
        qe, e = _irregular(q, rng)
        for parts in ENVS:
            monkeypatch.setenv("TSKV_PARTS", parts)
            check_vs_exact(engine, pages, truth, qe, e, "%s %s parts=%s" % (kind, name, parts), extra)
    pages.close()


@pytest.mark.parametrize("step,kind", ea.TB_CASES)
def test_tombstones(engine, step, kind):
    arena, descs, truth = ea.tombstone_arena(step, kind)
    tombs = ea.tombstone_list(truth, step)
    pages = engine.upload_pages(arena, descs)
    pages.set_tombstones(tombs)
    rng = np.random.default_rng(6)
    for name, q, extra in ea.tombstone_queries(truth, step):
        if q.width <= 0 or "slide" in extra:
            continue
        qe, e = _irregular(q, rng)
        check_vs_exact(engine, pages, truth, qe, e, "%d %s %s" % (step, kind, name), extra, tombstones=tombs)
    pages.close()


@pytest.mark.parametrize("tombstoned", [False, True])
def test_overlap_merge(engine, tombstoned):
    arena, descs, truth, files = ea.merge_arena()
    tombs = ea.merge_tombstones(truth) if tombstoned else None
    pages = engine.upload_pages(arena, descs)
    pages.set_chunk_files(files)
    if tombstoned:
        pages.set_tombstones(tombs)
    rng = np.random.default_rng(7)
    for name, q, extra in ea.merge_queries(truth):
        if q.width <= 0:
            continue
        qe, e = _irregular(q, rng)
        check_vs_exact(engine, pages, truth, qe, e, "merge %s tombstones=%s" % (name, tombstoned), extra,
                       tombstones=tombs, files=files)
    pages.close()


# ---- 3. coarsening --------------------------------------------------------------------------------------------------
def test_coarsened_grid_equals_folded_buckets(engine, monkeypatch):
    arena, descs, truth, _ = paths_arena()
    pages = engine.upload_pages(arena, descs)
    fbs, nb = bucket_spec(*span(truth), 10_000)
    nb = -(-nb // 6) * 6
    q = make_query(FIELDS, ("count", "sum", "min", "max"), width=10_000, first_bucket_start=fbs, n_buckets=nb)
    for m in (2, 3, 6):
        qe, e = edge_query(q, grid_edges(q)[::m])
        for parts in ENVS:
            monkeypatch.setenv("TSKV_PARTS", parts)
            fine = engine.scan_aggregate(pages, q)
            got = engine.scan_aggregate(pages, qe, edges=e)
            for j, (col, agg) in enumerate(got.names):
                what = "m=%d parts=%s col %s %s" % (m, parts, col, agg)
                v, ok = fine.column(col, agg)
                v, ok = v.reshape(nb // m, m), ok.reshape(nb // m, m)
                g, gok = got.column(col, agg)
                g, gok = g[0], gok[0]
                assert (gok == ok.any(axis=1)).all(), what
                if agg == "count":
                    exp = v.sum(axis=1)
                elif agg == "sum" and got.phys[col] == cabi.TSKV_PT_F64:
                    exp = np.where(ok, v, 0.0).sum(axis=1)
                    assert np.allclose(g[gok], exp[gok], rtol=1e-12, atol=0), what
                    continue
                elif agg == "sum":
                    with np.errstate(over="ignore"):
                        exp = np.where(ok, v, 0).astype(v.dtype).sum(axis=1, dtype=v.dtype)
                elif agg == "min":
                    exp = np.array([r[o].min() if o.any() else 0 for r, o in zip(v, ok)], dtype=v.dtype)
                else:
                    exp = np.array([r[o].max() if o.any() else 0 for r, o in zip(v, ok)], dtype=v.dtype)
                assert (g[gok] == exp[gok]).all(), what
    pages.close()


# ---- 4. refusals --------------------------------------------------------------------------------------------------
def _layout_status(engine, pages, q, e, gids=None, n_groups=0):
    L = cabi.OutputLayout()
    qc = q.to_c()
    ep = None if e is None else np.ascontiguousarray(e, dtype=np.int64)
    gp = None if gids is None else np.ascontiguousarray(gids, dtype=np.uint32)
    return engine.lib.tskvgpu_query_output_layout_edges(pages.handle, C.byref(qc), None if ep is None else ep.ctypes.data,
                                                       None if gp is None else gp.ctypes.data, n_groups, C.byref(L))


def _prepare_status(engine, pages, q, e, gids=None, n_groups=0):
    qc = q.to_c()
    ep = None if e is None else np.ascontiguousarray(e, dtype=np.int64)
    gp = None if gids is None else np.ascontiguousarray(gids, dtype=np.uint32)
    h = C.c_void_p()
    st = engine.lib.tskvgpu_scan_prepare_edges(engine.ctx, pages.handle, C.byref(qc), None if ep is None else ep.ctypes.data,
                                               None if gp is None else gp.ctypes.data, n_groups, C.byref(h))
    if h.value:
        engine.lib.tskvgpu_scan_destroy(engine.ctx, h)
    return st


def test_refusals(engine):
    arena, descs, truth = random_arena(np.random.default_rng(3), n_series=129, n_points=50, fields=FIELDS)
    pages = engine.upload_pages(arena, descs)
    good = np.array([0, 1_020_000, 1_040_000, 1_060_000], dtype=np.int64)
    base, _ = edge_query(make_query(FIELDS, PLAIN), good)
    INV = cabi.TSKV_ERR_INVALID_ARG

    def variant(**kw):
        q = copy.copy(base)
        q._keep = None
        for k, v in kw.items():
            setattr(q, k, v)
        return q
    cases = [
        ("edges NULL", base, None, None, 0),
        ("n_buckets 0", variant(n_buckets=0), good[:1], None, 0),
        ("not increasing", base, np.array([0, 5, 5, 1_060_000]), None, 0),
        ("decreasing", base, np.array([0, 1_060_000, 5, 1_070_000]), None, 0),
        ("span 2^63", variant(n_buckets=2), np.array([I64_MIN, 0, 1]), None, 0),
        ("width", variant(width=20_000), good, None, 0),
        ("origin", variant(origin=1), good, None, 0),
        ("first_bucket_start", variant(first_bucket_start=1), good, None, 0),
        ("group id >= n_groups", base, good, np.full(129, 3, np.uint32), 3),
        ("n_groups 0", base, good, np.zeros(129, np.uint32), 0),
        ("group map with group_by_series", variant(group_by_series=True), good, np.zeros(129, np.uint32), 1),
        ("cells > TSKV_MAX_GROUPED_CELLS", base, good, np.zeros(129, np.uint32), 2**31),
    ]
    for what, q, e, gids, ng in cases:
        assert _layout_status(engine, pages, q, e, gids, ng) == INV, what
        assert _prepare_status(engine, pages, q, e, gids, ng) == INV, what
    # the largest span is accepted
    q = variant(n_buckets=1)
    assert _layout_status(engine, pages, q, np.array([I64_MIN, -1])) == cabi.TSKV_OK
    with pytest.raises(ValueError):
        engine.prepare(pages, base, slide=10, edges=good)

    # FIRST / LAST key budget: yearly ns buckets leave 7 slot bits - 128 series pass, 129 are refused (the reference
    # predicts both); GROUP BY series needs no slot bits
    years = calendar_edges("year", 0, 3 * 365 * DAY)
    for n_series, gbs in ((128, False), (129, False), (129, True)):
        q, _ = edge_query(make_query(FIELDS, ALL_AGGS, series_ids=np.arange(n_series, dtype=np.uint32),
                                     group_by_series=gbs), years)
        try:
            exact_aggregate_edges(truth, q, years)
            err = None
        except ReferenceError as x:
            err = x.status
        st = _scan(engine, pages, q, edges=years)[1]
        assert st == err, (n_series, gbs, st, err)
        assert (err == cabi.TSKV_ERR_UNSUPPORTED) == (n_series == 129 and not gbs)
    pages.close()


@pytest.mark.parametrize("jitter", [0, 300])
def test_row_outside_the_edges(engine, jitter):
    """A selected row before edges[0] or at / after edges[n]: TSKV_ERR_BUCKET_RANGE naming a page of that row's series."""
    arena, descs, truth = random_arena(np.random.default_rng(4), n_series=40, n_points=300, fields=FIELDS, jitter=jitter)
    pages = engine.upload_pages(arena, descs)
    ts = {s: cgs[0][0] for s, cgs in truth.items()}
    lo = min(int(t.min()) for t in ts.values())
    hi = max(int(t.max()) for t in ts.values())
    low = min(ts, key=lambda s: int(ts[s].min()))
    high = max(ts, key=lambda s: int(ts[s].max()))
    for e, culprit in ((np.array([lo + 1, hi + 1]), low), (np.array([lo, lo + 1000, hi]), high)):
        for aggs in (PLAIN, ALL_AGGS):
            q, _ = edge_query(make_query(FIELDS, aggs), e)
            with pytest.raises(ReferenceError):
                exact_aggregate_edges(truth, q, e)
            with pytest.raises(TskvError) as err:
                engine.scan_aggregate(pages, q, edges=e)
            assert err.value.status == cabi.TSKV_ERR_BUCKET_RANGE
            assert 0 <= err.value.page < len(descs)
            page_series = int(descs[err.value.page]["series_id"])
            assert page_series in [s for s in ts if int(ts[s].min()) < e[0] or int(ts[s].max()) >= e[-1]], (page_series, culprit)
            # the same rows are fine once a time range leaves them out
            qr = copy.copy(q)
            qr.time_ranges, qr._keep = [(int(e[0]), int(e[-1]) - 1)], None
            check_vs_exact(engine, pages, truth, qr, e, "clipped %s %s" % (e, aggs))
    pages.close()


# ---- 5. two-shard exchange ------------------------------------------------------------------------------------------
def test_two_shard_exchange(engine):
    """Two series shards scanned separately with the same edges, their exchange regions concatenated like an
    all-gather and merged: every rank's result equals the exact reference over both shards."""
    import torch
    from cnosdb_b200.parallel import device_tensor
    arena, descs, truth = calendar_arena(3_000_000_000_000)
    e = calendar_edges("month", *span(truth))
    ids = np.arange(40, dtype=np.uint32)
    dev = torch.device("cuda", engine.device)
    for gbs in (False, True):
        q, _ = edge_query(make_query(FIELDS, ALL_AGGS, series_ids=ids, group_by_series=gbs, multi_rank=True), e)
        exp = exact_aggregate_edges(truth, q, e)
        scans, regions, keep = [], [], []
        for shard in (ids[ids % 2 == 0], ids[ids % 2 == 1]):
            pages = engine.upload_pages(arena, descs[np.isin(descs["series_id"], shard)])
            s = engine.prepare(pages, q, edges=e)
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


# ---- 6. graph replay ------------------------------------------------------------------------------------------------
def test_graph_replay(engine):
    arena, descs, truth = calendar_arena(0)
    pages = engine.upload_pages(arena, descs)
    e = calendar_edges("month", *span(truth))
    for aggs in (PLAIN, ALL_AGGS):
        q, _ = edge_query(make_query(FIELDS, aggs), e)
        once = engine.scan_aggregate(pages, q, edges=e)
        s = engine.prepare(pages, q, edges=e)
        for _ in range(4):  # the second enqueue captures the pass as a CUDA graph, the later ones replay it
            s.enqueue()
            s.sync()
            assert_same_result(s.finalize(), once, "graph replay %s" % (aggs,))
        s.close()
    pages.close()
