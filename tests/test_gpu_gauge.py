"""gauge_agg(time, x) (TSKV_QUERY_N_GAUGES) through the scan against tests/gauge_reference.py, bit for bit: RLE, jittered
and raw time pages with NULLs; bucketed, GROUP BY series, unbucketed, tag-group (ties of time across series), edge,
label and sliding grids; predicates, tombstones, host-resident pages with CRC on read; overlapping chunk files; integer
values that round in f64 and f64 specials; a query mixing every other operand kind; the multi-rank exchange at 1 / 3 /
4 / 8 ranks; repeated run / enqueue; every refusal."""
import ctypes as C

import numpy as np
import pytest

from cnosdb_b200 import cabi, datagen
from cnosdb_b200.engine import Engine, PushedAggregate, QueryOption, TskvError, sliding_window_grid
from tests.exact_arenas import two_file_arena
from tests.gauge_reference import cells_from_points, check_gauge, exact_gauge_cells, gauge_query_outputs, sliding_points
from tests.helpers import bucket_spec, random_arena
from tests.ranks import layouts, multi_rank, sharded_scans

pytestmark = pytest.mark.gpu

I64, U64, F64 = cabi.TSKV_PT_I64, cabi.TSKV_PT_U64, cabi.TSKV_PT_F64
T0, STEP, W = 1_000_000, 1000, 50_000
FIELDS = ((1, I64), (2, F64), (3, U64))
GAUGES = [PushedAggregate(c, pt, ["gauge_agg"]) for c, pt in FIELDS]


@pytest.fixture(scope="module")
def eng():
    e = Engine(0)
    yield e
    e.close()


def arena(seed, null_frac=0.2, jitter=0, raw_frac=0.0, n_series=24, n_points=400, fields=FIELDS, step=STEP):
    rng = np.random.default_rng(seed)
    return random_arena(rng, n_series=n_series, n_points=n_points, fields=fields, null_frac=null_frac, t0=T0, step=step,
                        jitter=jitter, raw_frac=raw_frac, multi_cg=True)


def grid_query(truth, columns=GAUGES, **kw):
    t_hi = max(int(ts[-1]) for cgs in truth.values() for ts, _ in cgs if len(ts))
    kw.setdefault("width", W)
    fbs, nb = bucket_spec(T0 - 10 * STEP, t_hi + STEP, kw["width"]) if kw["width"] > 0 else (0, 1)
    return QueryOption(list(columns), first_bucket_start=fbs, n_buckets=nb, **kw)


def check_gauges(res, truth, q, what, **kw):
    n_cells = res.n_groups * res.n_buckets
    gs = [c for c in q.columns if c.gauge_agg]
    starts = gauge_query_outputs(q)
    assert len(starts) == len(gs)
    seen = False
    for j0, c in zip(starts, gs):
        exact = exact_gauge_cells(truth, q, c.column_id, c.phys_type, n_cells, **kw)
        check_gauge(res, j0, exact, what="%s col %d" % (what, c.column_id))
        seen |= bool(exact[1][1].any())
    assert seen, what


@pytest.mark.parametrize("kind", ["rle", "jitter", "raw"])
def test_groupings(eng, kind):
    a, d, truth = arena(1, jitter=300 if kind == "jitter" else 0, raw_frac=0.5 if kind == "raw" else 0.0)
    pages = eng.upload_pages(a, d)
    try:
        sel = np.arange(0, 24, 2, dtype=np.uint32)
        q = grid_query(truth, series_ids=sel)
        check_gauges(eng.scan_aggregate(pages, q), truth, q, kind + " bucket")
        qs = grid_query(truth, series_ids=sel, group_by_series=True)
        check_gauges(eng.scan_aggregate(pages, qs), truth, qs, kind + " series")
        qu = grid_query(truth, width=0, time_ranges=[(T0 + 20 * STEP, T0 + 150 * STEP), (T0 + 300 * STEP, T0 + 900 * STEP)])
        check_gauges(eng.scan_aggregate(pages, qu), truth, qu, kind + " unbucketed, two ranges")
        gids = (sel % 3).astype(np.uint32)
        check_gauges(eng.scan_aggregate(pages, q, group_ids=gids, n_groups=3), truth, q, kind + " tags", group_ids=gids)
        edges = np.array([T0 - 10 * STEP, T0 + 77 * STEP, T0 + 200 * STEP, T0 + 555 * STEP, T0 + 2000 * STEP], dtype=np.int64)
        qe = grid_query(truth, width=0, series_ids=sel)
        qe.n_buckets = 4
        check_gauges(eng.scan_aggregate(pages, qe, edges=edges), truth, qe, kind + " edges", edges=edges)
        labels = np.array([1, 0, 1, 0], dtype=np.uint32)
        ql = grid_query(truth, width=0, series_ids=sel)
        ql.n_buckets = 2
        check_gauges(eng.scan_aggregate(pages, ql, edges=edges, labels=labels), truth, ql, kind + " labels", edges=edges,
                     labels=labels)
    finally:
        pages.close()


@pytest.mark.parametrize("window,slide", [(W, W // 5), (W, W), (30_000, 20_000), (W, 7_000), (20_000, 3_000)])
def test_sliding_windows(eng, window, slide):
    a, d, truth = arena(4, n_series=10, n_points=200)
    pages = eng.upload_pages(a, d)
    try:
        k = -(-window // slide)
        t_hi = max(int(ts[-1]) for cgs in truth.values() for ts, _ in cgs if len(ts))
        fbs = (T0 // slide) * slide - (k - 1) * slide - slide
        nb = (t_hi - fbs) // slide + 2
        for kw, groups in ((dict(), None), (dict(group_by_series=True), None), (dict(series_ids=np.arange(10, dtype=np.uint32)), "tags")):
            q = QueryOption(GAUGES, width=window, origin=0, first_bucket_start=fbs, n_buckets=nb, **kw)
            gids = (np.arange(10) % 3).astype(np.uint32) if groups else None
            res = eng.scan_aggregate(pages, q, slide=slide, group_ids=gids, n_groups=3 if groups else None)
            n_cells = res.n_groups * res.n_buckets
            for j0, c in zip(gauge_query_outputs(q), GAUGES):
                pts = sliding_points(truth, q, c.column_id, c.phys_type, slide, res.n_groups,
                                     **({"group_ids": gids} if groups else {}))
                check_gauge(res, j0, cells_from_points(pts, n_cells), what="sliding %d/%d %s" % (window, slide, kw))
    finally:
        pages.close()


def tie_arena():
    """Four series with the same timestamps (ties of time across series in one tag group), values that round in f64."""
    b = datagen.ArenaBuilder()
    truth = {}
    rng = np.random.default_rng(9)
    for sid in range(4):
        ts = T0 + np.arange(120, dtype=np.int64) * STEP
        iv = (rng.integers(-(2**62), 2**62, ts.size) | 1).astype(np.int64) * 2 + 1
        uv = rng.integers(2**63, 2**64 - 1, ts.size, dtype=np.uint64) | np.uint64(1)
        fv = rng.choice(np.array([0.0, -0.0, np.inf, -np.inf, 1.5, np.nan], dtype=np.float64), ts.size)
        fv = fv.view(np.uint64).copy()
        fv[::7] = 0x7FF8000000000123  # a NaN payload
        fv = fv.view(np.float64)
        valid = rng.random(ts.size) >= 0.2
        cols = {1: (iv, valid), 2: (fv, valid.copy()), 3: (uv, valid.copy())}
        b.add_column_group(sid, ts, [(c, pt, cols[c][0], cols[c][1], None) for c, pt in FIELDS])
        truth[sid] = [(ts, cols)]
    arena_, descs = b.finish()
    return arena_, descs, truth


def test_ties_rounding_and_specials(eng):
    a, d, truth = tie_arena()
    pages = eng.upload_pages(a, d)
    try:
        for kw in (dict(), dict(width=0), dict(group_by_series=True), dict(width=STEP * 7)):
            q = grid_query(truth, **kw)
            check_gauges(eng.scan_aggregate(pages, q), truth, q, "ties %s" % kw)
        q = grid_query(truth)
        gids = np.array([0, 1, 0, 1], dtype=np.uint32)
        check_gauges(eng.scan_aggregate(pages, q, group_ids=gids, n_groups=2), truth, q, "tie tags", group_ids=gids)
    finally:
        pages.close()


def test_filters_tombstones_host_resident(eng):
    a, d, truth = arena(2)
    tombs = cabi.tombstones([(3, 2, T0 + 50 * STEP, T0 + 120 * STEP), (5, 1, T0, T0 + 300 * STEP),
                             (7, None, T0 + 10 * STEP, T0 + 40 * STEP), (None, None, T0 + 600 * STEP, T0 + 610 * STEP)])
    for host in (False, True):
        pages = eng.upload_pages(a, d, host_resident=host, verify_on_read=True)
        try:
            pages.set_tombstones(tombs)
            q = grid_query(truth, predicates=[(1, I64, ">", -40), (2, F64, "<=", 30.0)],
                           time_ranges=[(T0 + 5 * STEP, T0 + 800 * STEP)], group_by_series=True)
            check_gauges(eng.scan_aggregate(pages, q), truth, q, "filters host=%s" % host, tombstones=tombs)
        finally:
            pages.close()


def test_overlapping_chunk_files(eng):
    a, d, truth, files, _ = two_file_arena(T0, STEP)
    pages = eng.upload_pages(a, d)
    try:
        pages.set_chunk_files(files)
        for gbs in (True, False):
            q = grid_query(truth, columns=GAUGES[:2], group_by_series=gbs)
            check_gauges(eng.scan_aggregate(pages, q), truth, q, "overlap gbs=%s" % gbs, files=files)
    finally:
        pages.close()


def test_mixed_query_outputs_and_counters(eng):
    """Gauges on top of projected aggregates, a pair, a median, an increase, a mode and a distinct: the other outputs equal
    those of the query without gauges, and the counters equal those of the query with the operands as COUNT columns."""
    a, d, truth = arena(3)
    pages = eng.upload_pages(a, d)
    try:
        base = [PushedAggregate(1, I64, ["count", "sum", "min", "max", "median", "mode"]),
                PushedAggregate(2, F64, ["count", "increase", "count_distinct"])]
        extra = [PushedAggregate(1, I64, ["gauge_agg"]), PushedAggregate(3, U64, ["gauge_agg"]), PushedAggregate(2, F64, ["gauge_agg"])]
        kw = dict(pairs=[(1, I64, 2, F64)], predicates=[(3, U64, ">=", 0)], group_by_series=True)
        q = grid_query(truth, columns=base + extra, **kw)
        r = eng.scan_aggregate(pages, q)
        c = eng.counters()
        q0 = grid_query(truth, columns=base, **kw)
        r0 = eng.scan_aggregate(pages, q0)
        for j0, name in enumerate(q0.output_names()):
            j = r.names.index(name)
            np.testing.assert_array_equal(r.validity[j], r0.validity[j0], err_msg=str(name))
            ok = r.validity[j]
            x, y = r.values[j][ok], r0.values[j0][ok]
            if name[1] in ("c", "m2x", "m2y", "increase") or (name[1] in ("sum", "mean") and r.phys.get(name[0]) == F64):
                np.testing.assert_allclose(x.view(np.float64), y.view(np.float64), rtol=1e-12, atol=1e-300, err_msg=str(name))
            else:
                np.testing.assert_array_equal(x, y, err_msg=str(name))
        check_gauges(r, truth, q, "mixed")
        qc = grid_query(truth, columns=base + [PushedAggregate(3, U64, ["count"])], **kw)
        eng.scan_aggregate(pages, qc)
        cc = eng.counters()
        for k in ("page_read_count", "page_read_bytes", "points_decoded", "rows_in_range", "pruned_page_count"):
            assert c[k] == cc[k], k
        assert c["kernel_launches"] > cc["kernel_launches"]
    finally:
        pages.close()


@pytest.mark.parametrize("n", [1, 3, 4, 8])
def test_ranks(eng, n):
    a, d, truth = arena(7, n_series=16, n_points=200)
    ids = np.arange(16, dtype=np.uint32)
    pages = eng.upload_pages(a, d)
    try:
        for kw in (dict(), dict(group_by_series=True), dict(width=0)):
            q = multi_rank(grid_query(truth, series_ids=ids, **kw))
            whole = eng.scan_aggregate(pages, q)
            check_gauges(whole, truth, q, "whole %s" % kw)
            for name, (shards, order) in layouts(ids, n).items():
                for r in sharded_scans(eng, a, d, q, shards, order=order):
                    for j in range(len(whole.names)):
                        np.testing.assert_array_equal(r.validity[j], whole.validity[j], err_msg="%d %s" % (n, name))
                        if whole.names[j][1].startswith("gauge_"):
                            np.testing.assert_array_equal(r.values[j], whole.values[j], err_msg="%d %s %s" % (n, name, whole.names[j]))
    finally:
        pages.close()


def test_repeated_run_and_enqueue(eng):
    a, d, truth = arena(6)
    t_hi = max(int(ts[-1]) for cgs in truth.values() for ts, _ in cgs if len(ts))
    for slide in (None, W // 5):
        q = grid_query(truth, group_by_series=True)
        if slide:
            q.first_bucket_start, q.n_buckets = sliding_window_grid(T0, t_hi, W, slide)
        pages = eng.upload_pages(a, d)
        try:
            s = eng.prepare(pages, q, slide=slide) if slide else eng.prepare(pages, q)
            try:
                s.run()
                first = s.finalize()
                if not slide:
                    check_gauges(first, truth, q, "run")
                for _ in range(3):
                    s.enqueue()
                    s.sync()
                    r = s.finalize()
                    np.testing.assert_array_equal(r.values, first.values)
                    np.testing.assert_array_equal(r.validity, first.validity)
            finally:
                s.close()
        finally:
            pages.close()


class _RawQuery(QueryOption):
    def __init__(self, *a, patch=None, flags=0, **kw):
        super().__init__(*a, **kw)
        self.patch, self.flags = patch, flags

    def to_c(self):
        q = super().to_c()
        if self.patch:
            self.patch(q.columns[len(self.projected()) + cabi.query_n_gauges(q.reserved) - 1])
        q.reserved |= self.flags
        return q


def test_refusals(eng):
    a, d, truth = arena(5, n_series=4, n_points=50)
    pages = eng.upload_pages(a, d)
    try:
        def status(q, **kw):
            try:
                eng.scan_aggregate(pages, q, **kw)
            except TskvError as e:
                return e.status
            return cabi.TSKV_OK

        def prepare_status(q):
            h = C.c_void_p()
            cq = q.to_c()
            st = eng.lib.tskvgpu_scan_prepare(eng.ctx, pages.handle, C.byref(cq), C.byref(h))
            if h.value:
                eng.lib.tskvgpu_scan_destroy(eng.ctx, h)
            return st
        INV, UNS = cabi.TSKV_ERR_INVALID_ARG, cabi.TSKV_ERR_UNSUPPORTED
        op = lambda cid=1, pt=I64: PushedAggregate(cid, pt, ["gauge_agg"])
        assert status(grid_query(truth, columns=[op()] * 8)) == cabi.TSKV_OK
        assert status(grid_query(truth, columns=[op()] * 9)) == INV
        assert status(grid_query(truth, columns=[op(5, cabi.TSKV_PT_BOOL)])) == INV
        assert status(grid_query(truth, columns=[op(0, cabi.TSKV_PT_TIME)])) == INV
        assert status(grid_query(truth, columns=[op(1, 9)])) == INV
        assert status(grid_query(truth, columns=[PushedAggregate(1, I64, ["count"]), op(1, F64)])) == INV
        assert status(grid_query(truth, columns=[op(1, I64), op(1, U64)])) == INV
        many = lambda n: [PushedAggregate(100 + i, I64, ["count"]) for i in range(n)] + [op()] * 8
        assert status(grid_query(truth, columns=many(118))) == cabi.TSKV_OK
        assert status(grid_query(truth, columns=many(119))) == INV
        masked = _RawQuery([op()], first_bucket_start=0, n_buckets=1, patch=lambda c: setattr(c, "agg_mask", cabi.TSKV_AGG_COUNT))
        assert prepare_status(masked) == INV
        assert prepare_status(_RawQuery([op()], first_bucket_start=0, n_buckets=1, flags=cabi.TSKV_QUERY_MULTI_RANK)) == INV
        s = eng.prepare(pages, grid_query(truth, columns=[op()]))
        try:
            s.run()
            with pytest.raises(TskvError) as e:
                s.partials()
            assert e.value.status == UNS
        finally:
            s.close()
    finally:
        pages.close()


@pytest.mark.parametrize("time_enc", ["raw", "delta"])
def test_null_time_pages(eng, time_enc):
    """Time pages that mark rows NULL (raw and delta encoded): those rows are not selected, and the lane carries its
    timestamp cursor across them."""
    rng = np.random.default_rng(13)
    b = datagen.ArenaBuilder()
    truth = {}
    enc_t = datagen.encode_raw if time_enc == "raw" else datagen.encode_timestamps
    dt = {I64: np.int64, U64: np.uint64, F64: np.float64}
    for sid in range(4):
        cgs = []
        for k in range(3):
            n = 80
            ts = T0 + (np.arange(n, dtype=np.int64) + 100 * k) * STEP
            if time_enc == "delta":  # jittered: a simple8b time page
                ts = ts + rng.integers(0, 300, n)
            tvalid = rng.random(n) > 0.2
            tvalid[0] = k != 1  # a page whose first row has a NULL time
            cols = {}
            tvals = ts[tvalid]
            if time_enc == "delta" and not tvalid[0]:  # a NULL row 0 of a simple8b time page swallows its first value
                tvals = np.concatenate([tvals[:1] - 500, tvals])
            b.add_page(datagen.build_page(enc_t(tvals), n, tvalid), sid, 0, cabi.TSKV_PT_TIME, n)
            for cid, pt in FIELDS:
                v = rng.integers(-50, 50, n).astype(dt[pt]) if pt != U64 else rng.integers(0, 50, n).astype(np.uint64)
                valid = rng.random(n) > 0.1
                kept = v[valid].view(np.int64) if pt == U64 else v[valid]
                enc = datagen.encode_floats if pt == F64 else datagen.encode_integers
                b.add_page(datagen.build_page(enc(kept), n, valid), sid, cid, pt, n)
                cols[cid] = (v, valid & tvalid)
            cgs.append((ts, cols))
        truth[sid] = cgs
    a, d = b.finish()
    pages = eng.upload_pages(a, d)
    try:
        for kw in (dict(group_by_series=True), dict(), dict(width=0)):
            q = grid_query(truth, **kw)
            check_gauges(eng.scan_aggregate(pages, q), truth, q, "NULL-time pages %s %s" % (time_enc, kw))
    finally:
        pages.close()


@pytest.mark.parametrize("n", [3, 8])
def test_ranks_sliding_and_tags(eng, n):
    """The exchange after the pane fold (sliding windows) and across tag groups whose series tie in time (the global
    slot breaks the tie on every rank): every layout equals the single-rank scan."""
    for arena_of, shape in ((lambda: arena(7, n_series=16, n_points=200), "random"), (tie_arena, "ties")):
        a, d, truth = arena_of()
        ids = np.array(sorted(truth), dtype=np.uint32)
        t_hi = max(int(ts[-1]) for cgs in truth.values() for ts, _ in cgs if len(ts))
        pages = eng.upload_pages(a, d)
        try:
            fbs, nb = sliding_window_grid(T0, t_hi, W, W // 5)
            qs = multi_rank(QueryOption(GAUGES, series_ids=ids, width=W, first_bucket_start=fbs, n_buckets=nb))
            gids = (np.arange(ids.size) % 2).astype(np.uint32)
            qt = multi_rank(grid_query(truth, series_ids=ids))
            for q, prep, what in ((qs, dict(slide=W // 5), "sliding"), (qt, dict(group_ids=gids, n_groups=2), "tags")):
                whole = eng.scan_aggregate(pages, q, **prep)
                if what == "tags":
                    check_gauges(whole, truth, q, "%s whole tags" % shape, group_ids=gids)
                for name, (shards, order) in layouts(ids, min(n, ids.size)).items():
                    for r in sharded_scans(eng, a, d, q, shards, order=order, **prep):
                        for j in range(len(whole.names)):
                            if whole.names[j][1].startswith("gauge_"):
                                np.testing.assert_array_equal(r.validity[j], whole.validity[j], err_msg="%s %d %s" % (what, n, name))
                                np.testing.assert_array_equal(r.values[j], whole.values[j], err_msg="%s %d %s %s" % (what, n, name, whole.names[j]))
        finally:
            pages.close()
