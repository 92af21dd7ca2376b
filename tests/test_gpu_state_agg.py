"""compact_state_agg(time, x) (TSKV_QUERY_N_STATE_AGGS) through the scan against tests/state_agg_reference.py, compared as
maps: one-series ungrouped, GROUP BY series, one-series tag groups and edge grids; row-drop and column tombstones (the
latter make NULL states); predicates; overlapping chunk files; NULL-time pages; host-resident and verify-on-read page
sets; u64 states above 2^63; a replay of the prepared scan, byte for byte; every refusal."""
import ctypes as C

import numpy as np
import pytest

from cnosdb_b200 import cabi, datagen
from cnosdb_b200.engine import Engine, PushedAggregate, QueryOption, TskvError, duration_in
from tests.exact_arenas import two_file_arena
from tests.helpers import bucket_spec
from tests.state_agg_reference import check_state_maps, exact_state_maps

pytestmark = pytest.mark.gpu

I64, U64, F64 = cabi.TSKV_PT_I64, cabi.TSKV_PT_U64, cabi.TSKV_PT_F64
T0, STEP, W = 1_000_000, 1000, 50_000
FIELDS = ((1, I64), (3, U64))
STATES = [PushedAggregate(c, pt, ["compact_state_agg"]) for c, pt in FIELDS]


@pytest.fixture(scope="module")
def eng():
    e = Engine(0)
    yield e
    e.close()


def run_values(rng, n, pt, mean_run=6):
    """n states in runs of about mean_run rows: i64 from a small signed set, u64 around and above 2^63."""
    pool = (np.array([-(2**63), -7, 0, 3, 2**63 - 1], dtype=np.int64) if pt == I64 else
            np.array([0, 5, 2**63 - 1, 2**63, 2**64 - 1], dtype=np.uint64))
    out = np.empty(n, dtype=pool.dtype)
    i = 0
    while i < n:
        k = int(rng.geometric(1.0 / mean_run))
        out[i:i + k] = pool[rng.integers(0, pool.size)]
        i += k
    return out


def state_arena(seed, n_series=8, n_points=300, null_frac=0.15, jitter=0, raw_frac=0.0, mean_run=6):
    """Series of one to three column groups back to back in time, fields FIELDS with runs of states and NULLs."""
    rng = np.random.default_rng(seed)
    b = datagen.ArenaBuilder()
    truth = {}
    for sid in range(n_series):
        t_start = T0
        for _ in range(int(rng.integers(1, 4))):
            n = int(rng.integers(1, n_points + 1))
            ts = t_start + np.arange(n, dtype=np.int64) * STEP
            if jitter:
                ts = ts + rng.integers(0, jitter + 1, n)
            t_start = int(ts[-1]) + STEP
            fl, cols = [], {}
            for col, pt in FIELDS:
                v = run_values(rng, n, pt, mean_run)
                valid = rng.random(n) >= null_frac
                enc = datagen.encode_raw if raw_frac and rng.random() < raw_frac else None
                fl.append((col, pt, v, valid, enc))
                cols[col] = (v, valid)
            b.add_column_group(sid, ts, fl)
            truth.setdefault(sid, []).append((ts, cols))
    a, d = b.finish()
    return a, d, truth


def t_hi_of(truth):
    return max(int(ts[-1]) for cgs in truth.values() for ts, _ in cgs if len(ts))


def grid_query(truth, columns=STATES, **kw):
    kw.setdefault("width", W)
    fbs, nb = bucket_spec(T0 - 10 * STEP, t_hi_of(truth) + 2 * STEP, kw["width"]) if kw["width"] > 0 else (0, 1)
    return QueryOption(list(columns), first_bucket_start=fbs, n_buckets=nb, **kw)


def check(res, truth, q, what, **kw):
    n_cells = res.n_groups * res.n_buckets
    seen = 0
    for cid, pt in q.state_aggs():
        exact = exact_state_maps(truth, q, cid, pt, n_cells, **kw)
        check_state_maps(res, cid, exact, "%s col %d" % (what, cid))
        seen += sum(len(m) for m in exact)
    assert seen, what


@pytest.mark.parametrize("kind", ["rle", "jitter", "raw"])
def test_groupings(eng, kind):
    a, d, truth = state_arena(1, jitter=300 if kind == "jitter" else 0, raw_frac=0.5 if kind == "raw" else 0.0)
    pages = eng.upload_pages(a, d)
    try:
        for sid in (0, 5):
            one = np.array([sid], dtype=np.uint32)
            q = grid_query(truth, series_ids=one)
            check(eng.scan_aggregate(pages, q), truth, q, "%s one series %d" % (kind, sid))
            qu = grid_query(truth, width=0, series_ids=one, time_ranges=[(T0 + 20 * STEP, T0 + 150 * STEP), (T0 + 300 * STEP, T0 + 900 * STEP)])
            check(eng.scan_aggregate(pages, qu), truth, qu, "%s unbucketed %d" % (kind, sid))
        qs = grid_query(truth, group_by_series=True)
        check(eng.scan_aggregate(pages, qs), truth, qs, kind + " by series")
        sel = np.arange(0, 8, 2, dtype=np.uint32)
        gids = np.array([2, 0, 3, 1], dtype=np.uint32)  # one series per tag group
        qt = grid_query(truth, series_ids=sel)
        check(eng.scan_aggregate(pages, qt, group_ids=gids, n_groups=4), truth, qt, kind + " tags", group_ids=gids)
        edges = np.array([T0 - 10 * STEP, T0 + 77 * STEP, T0 + 200 * STEP, T0 + 555 * STEP, T0 + 2000 * STEP], dtype=np.int64)
        qe = grid_query(truth, width=0, group_by_series=True)
        qe.n_buckets = 4
        check(eng.scan_aggregate(pages, qe, edges=edges), truth, qe, kind + " edges", edges=edges)
    finally:
        pages.close()


def test_filters_tombstones_host_resident(eng):
    a, d, truth = state_arena(2)
    tombs = cabi.tombstones([(3, 1, T0 + 50 * STEP, T0 + 120 * STEP), (5, 3, T0, T0 + 300 * STEP),
                             (7, None, T0 + 10 * STEP, T0 + 40 * STEP), (None, None, T0 + 600 * STEP, T0 + 610 * STEP)])
    for host, verify in ((False, False), (False, True), (True, True)):
        pages = eng.upload_pages(a, d, host_resident=host, verify_on_read=verify)
        try:
            pages.set_tombstones(tombs)
            q = grid_query(truth, predicates=[(1, I64, ">", -8)], time_ranges=[(T0 + 5 * STEP, T0 + 800 * STEP)],
                           group_by_series=True)
            check(eng.scan_aggregate(pages, q), truth, q, "filters host=%s" % host, tombstones=tombs)
            q0 = grid_query(truth, group_by_series=True, width=0)
            r = eng.scan_aggregate(pages, q0)
            check(r, truth, q0, "tombstones only host=%s" % host, tombstones=tombs)
            # a column tombstone makes NULL states: series 5's column 3 from its first row on
            assert None in r.state_maps(3)[5][0]
        finally:
            pages.close()


def test_overlapping_chunk_files(eng):
    a, d, truth, files, _ = two_file_arena(T0, STEP)
    pages = eng.upload_pages(a, d)
    try:
        pages.set_chunk_files(files)
        col = [PushedAggregate(1, I64, ["compact_state_agg"])]
        for kw in (dict(group_by_series=True), dict(group_by_series=True, width=7 * STEP), dict(series_ids=np.array([2], np.uint32))):
            q = grid_query(truth, columns=col, **kw)
            check(eng.scan_aggregate(pages, q), truth, q, "overlap %s" % kw, files=files)
    finally:
        pages.close()


def test_null_time_pages(eng):
    """Raw time pages that mark rows NULL: those rows are skipped (evaluate skips NULL times); NULL values are states."""
    rng = np.random.default_rng(9)
    b = datagen.ArenaBuilder()
    truth = {}
    for sid in range(4):
        cgs = []
        for k in range(3):
            n = 80
            ts = T0 + (np.arange(n, dtype=np.int64) + 100 * k) * STEP
            tvalid = rng.random(n) > 0.2
            fields, cols = [], {}
            for cid, pt in FIELDS:
                v = run_values(rng, n, pt)
                valid = rng.random(n) > 0.2
                fields.append((cid, pt, v, valid))
                cols[cid] = (v, valid)
            b.add_page(datagen.build_page(datagen.encode_raw(ts[tvalid]), n, tvalid), sid, 0, cabi.TSKV_PT_TIME, n)
            for cid, pt, v, valid in fields:
                kept = v[valid].view(np.int64) if pt == U64 else v[valid]
                b.add_page(datagen.build_page(datagen.encode_integers(kept), n, valid), sid, cid, pt, n)
            cgs.append((ts[tvalid], {c: (v[tvalid], ok[tvalid]) for c, (v, ok) in cols.items()}))
        truth[sid] = cgs
    a, d = b.finish()
    pages = eng.upload_pages(a, d)
    try:
        q = grid_query(truth, group_by_series=True)
        check(eng.scan_aggregate(pages, q), truth, q, "NULL-time pages")
    finally:
        pages.close()


def test_u64_states_above_2_63_and_duration_in(eng):
    b = datagen.ArenaBuilder()
    ts = T0 + np.arange(6, dtype=np.int64) * STEP
    u = np.array([2**64 - 1, 2**63, 2**63, 5, 2**64 - 1, 0], dtype=np.uint64)
    i = np.array([-(2**63), 2**63 - 1, -1, -1, 0, -(2**63)], dtype=np.int64)
    valid = np.array([1, 1, 0, 1, 1, 1], dtype=bool)
    b.add_column_group(0, ts, [(1, I64, i, valid, None), (3, U64, u, valid, None)])
    a, d = b.finish()
    truth = {0: [(ts, {1: (i, valid), 3: (u, valid)})]}
    pages = eng.upload_pages(a, d)
    try:
        q = grid_query(truth, width=0)
        r = eng.scan_aggregate(pages, q)
        check(r, truth, q, "extremes")
        mu = r.state_maps(3)[0][0]
        assert list(mu) == [None, 0, 5, 2**63, 2**64 - 1]  # NULL first, then unsigned order
        assert mu == {None: STEP, 0: 0, 5: STEP, 2**63: STEP, 2**64 - 1: 2 * STEP}
        mi = r.state_maps(1)[0][0]
        assert list(mi) == [None, -(2**63), -1, 0, 2**63 - 1]  # then signed order
        assert duration_in(mi, -(2**63)) == STEP and duration_in(mi, 12345) == 0 and duration_in(mi, None) == STEP
    finally:
        pages.close()


def test_prepared_replay_is_byte_identical(eng):
    a, d, truth = state_arena(6)
    pages = eng.upload_pages(a, d)
    try:
        q = grid_query(truth, group_by_series=True, width=7 * STEP)
        s = eng.prepare(pages, q)
        try:
            off, states, valid, durs = s.state_durations(0)  # before the first run: empty maps
            assert not off.any() and states.size == valid.size == durs.size == 0
            s.run()
            first = s.finalize()
            check(first, truth, q, "prepared")
            csr = [s.state_durations(k) for k in range(2)]
            for _ in range(3):
                s.enqueue()
                s.sync()
                r = s.finalize()
                np.testing.assert_array_equal(r.values, first.values)
                np.testing.assert_array_equal(r.validity, first.validity)
                for k in range(2):
                    for x, y in zip(s.state_durations(k), csr[k]):
                        assert x.dtype == y.dtype and x.tobytes() == y.tobytes()
        finally:
            s.close()
    finally:
        pages.close()


def test_caller_bounds_without_time_span(eng):
    """Time bounds handed in by the caller that give a group with rows min > max: the records are sized for one piece
    per row there, and the maps stay exact."""
    a, d, truth = state_arena(8, n_points=400)
    bounds = np.array([(int(ts[0]), int(ts[-1])) for sid in truth for ts, _ in truth[sid]], dtype=np.int64)
    bounds[::2] = (1, 0)
    pages = eng.upload_pages(a, d)
    try:
        pages.set_time_bounds(bounds)
        q = grid_query(truth, group_by_series=True, width=3 * STEP)
        check(eng.scan_aggregate(pages, q), truth, q, "caller bounds with min > max")
    finally:
        pages.close()


def test_mixed_query_outputs(eng):
    """State aggs on top of projected aggregates, a median, a mode and a gauge: the other outputs equal those of the query
    without state aggs, and the counters those of the query with the operands as COUNT columns."""
    a, d, truth = state_arena(3)
    pages = eng.upload_pages(a, d)
    try:
        base = [PushedAggregate(1, I64, ["count", "sum", "min", "max", "median", "mode", "gauge_agg"]),
                PushedAggregate(3, U64, ["count", "increase"])]
        kw = dict(group_by_series=True)
        q = grid_query(truth, columns=base + STATES, **kw)
        r = eng.scan_aggregate(pages, q)
        c = eng.counters()
        q0 = grid_query(truth, columns=base, **kw)
        r0 = eng.scan_aggregate(pages, q0)
        for j0, name in enumerate(q0.output_names()):
            j = r.names.index(name)
            np.testing.assert_array_equal(r.validity[j], r0.validity[j0], err_msg=str(name))
            np.testing.assert_array_equal(r.values[j][r.validity[j]], r0.values[j0][r0.validity[j0]], err_msg=str(name))
        check(r, truth, q, "mixed")
        eng.scan_aggregate(pages, q0)
        cc = eng.counters()
        for k in ("page_read_count", "page_read_bytes", "points_decoded", "rows_in_range", "pruned_page_count"):
            assert c[k] == cc[k], k
    finally:
        pages.close()


class _RawQuery(QueryOption):
    def __init__(self, *a, patch=None, flags=0, **kw):
        super().__init__(*a, **kw)
        self.patch, self.flags = patch, flags

    def to_c(self):
        q = super().to_c()
        if self.patch:
            self.patch(q.columns[len(self.projected())])
        q.reserved |= self.flags
        return q


def test_refusals(eng):
    a, d, truth = state_arena(5, n_series=4, n_points=50)
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
        op = lambda cid=1, pt=I64: PushedAggregate(cid, pt, ["compact_state_agg"])
        one = dict(series_ids=np.array([1], np.uint32))
        assert status(grid_query(truth, columns=[op()] * 7, **one)) == cabi.TSKV_OK
        assert status(grid_query(truth, columns=[op(2, F64)], **one)) == INV
        assert status(grid_query(truth, columns=[op(5, cabi.TSKV_PT_BOOL)], **one)) == INV
        assert status(grid_query(truth, columns=[op(0, cabi.TSKV_PT_TIME)], **one)) == INV
        assert status(grid_query(truth, columns=[PushedAggregate(1, I64, ["count"]), op(1, U64)], **one)) == INV
        many = lambda n: [PushedAggregate(100 + i, I64, ["count"]) for i in range(n)] + [op()] * 7
        assert status(grid_query(truth, columns=many(119), **one)) == cabi.TSKV_OK
        assert status(grid_query(truth, columns=many(120), **one)) == INV
        masked = _RawQuery([op()], first_bucket_start=0, n_buckets=1, patch=lambda c: setattr(c, "agg_mask", cabi.TSKV_AGG_COUNT), **one)
        assert prepare_status(masked) == INV
        # a cell that could hold two series: ungrouped over several, a tag group of two
        assert status(grid_query(truth)) == UNS
        assert status(grid_query(truth, series_ids=np.array([0, 1], np.uint32)), group_ids=np.array([0, 0], np.uint32), n_groups=1) == UNS
        qs = grid_query(truth, group_by_series=True)
        assert status(qs, slide=W // 5) == UNS
        edges = np.array([T0 - 10 * STEP, T0 + 77 * STEP, T0 + 200 * STEP], dtype=np.int64)
        ql = grid_query(truth, width=0, group_by_series=True)
        ql.n_buckets = 1
        assert status(ql, edges=edges, labels=np.array([0, 0], np.uint32)) == UNS
        assert prepare_status(_RawQuery([op()], first_bucket_start=0, n_buckets=1, flags=cabi.TSKV_QUERY_MULTI_RANK,
                                        series_ids=np.array([1], np.uint32))) == UNS
        # an unbucketed cell that can span 2^63: a time range as wide as the type
        b = datagen.ArenaBuilder()
        ts = np.array([-(2**62) * 2, 2**62, 2**63 - 1], dtype=np.int64)
        v = np.array([1, 2, 3], dtype=np.int64)
        b.add_column_group(0, ts, [(1, I64, v, None, datagen.encode_raw)])
        wa, wd = b.finish()
        wide = eng.upload_pages(wa, wd)
        try:
            with pytest.raises(TskvError) as e:
                eng.scan_aggregate(wide, QueryOption([op()], n_buckets=1))
            assert e.value.status == UNS
            r = eng.scan_aggregate(wide, QueryOption([op()], n_buckets=1, time_ranges=[(0, 2**63 - 1)]))
            assert r.state_maps(1)[0][0] == {2: 2**63 - 1 - 2**62, 3: 0}
        finally:
            wide.close()
        # a column group without a page of the operand
        b = datagen.ArenaBuilder()
        b.add_column_group(0, T0 + np.arange(4, dtype=np.int64) * STEP, [(1, I64, np.arange(4, dtype=np.int64), None, None)])
        b.add_column_group(0, T0 + np.arange(10, 14, dtype=np.int64) * STEP, [(3, U64, np.arange(4, dtype=np.uint64), None, None)])
        ma, md = b.finish()
        missing = eng.upload_pages(ma, md)
        try:
            with pytest.raises(TskvError) as e:
                eng.scan_aggregate(missing, QueryOption([op()], n_buckets=1))
            assert e.value.status == UNS
            r = eng.scan_aggregate(missing, QueryOption([op()], n_buckets=1, time_ranges=[(T0, T0 + 5 * STEP)]))
            assert r.state_maps(1)[0][0] == {0: STEP, 1: STEP, 2: STEP, 3: 0}
        finally:
            missing.close()
        s = eng.prepare(pages, grid_query(truth, columns=[op()], **one))
        try:
            s.run()
            for call in (s.partials, s.exchange_view):
                with pytest.raises(TskvError) as e:
                    call()
                assert e.value.status == UNS
            with pytest.raises(TskvError) as e:
                s.state_durations(1)
            assert e.value.status == INV
        finally:
            s.close()
    finally:
        pages.close()
