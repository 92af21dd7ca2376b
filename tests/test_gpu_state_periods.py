"""state_agg(time, x)'s periods (TSKV_STATE_PERIODS) through the scan against tests/state_periods_reference.py's joined
periods, exactly and in order: one-series ungrouped, GROUP BY series, one-series tag groups, tumbling and edge grids;
predicates, row-drop and column tombstones (NULL states), host-resident page sets; overlapping chunk files; NULL-time
pages; u64 states above 2^63; caller bounds without a time span; a replay byte for byte; empty lists before the first run;
a flagged and an unflagged operand in one query; a cell whose rows share one time. A query with the flag gives the
durations, outputs and counters of the same query without it. Every refusal."""
import copy
import ctypes as C

import numpy as np
import pytest

from cnosdb_b200 import cabi, datagen
from cnosdb_b200.engine import CompactAggError, Engine, PushedAggregate, QueryOption, TskvError, duration_in, state_at
from tests.exact_arenas import two_file_arena
from tests.state_agg_reference import check_state_maps, exact_state_maps
from tests.state_periods_reference import check_state_periods, exact_state_periods
from tests.test_gpu_state_agg import FIELDS, STEP, T0, W, _RawQuery, grid_query, run_values, state_arena

pytestmark = pytest.mark.gpu

I64, U64, F64 = cabi.TSKV_PT_I64, cabi.TSKV_PT_U64, cabi.TSKV_PT_F64
PERIODS = [PushedAggregate(c, pt, ["state_agg"]) for c, pt in FIELDS]
COUNTERS = ("page_read_count", "page_read_bytes", "points_decoded", "rows_in_range", "pruned_page_count")


@pytest.fixture(scope="module")
def eng():
    e = Engine(0)
    yield e
    e.close()


def compact(columns):
    """The same columns with every state_agg asked as compact_state_agg: the same operands without the flag."""
    out = []
    for c in columns:
        if c.state_agg:
            c = copy.copy(c)
            c.state_agg, c.compact_state_agg = False, True
        out.append(c)
    return out


def check(eng, pages, truth, q, what, **kw):
    """q's periods and maps against the reference; q without the flag gives the same outputs, maps and counters."""
    scan_kw = {k: kw[k] for k in ("group_ids", "edges") if k in kw}
    if "group_ids" in kw:
        scan_kw["n_groups"] = int(max(kw["group_ids"])) + 1
    r = eng.scan_aggregate(pages, q, **scan_kw)
    c1 = eng.counters()
    q0 = QueryOption(compact(q.columns), **{k: getattr(q, k) for k in ("series_ids", "time_ranges", "predicates", "width",
                                                                        "first_bucket_start", "n_buckets", "group_by_series")})
    r0 = eng.scan_aggregate(pages, q0, **scan_kw)
    c0 = eng.counters()
    np.testing.assert_array_equal(r.values, r0.values, err_msg=what)
    np.testing.assert_array_equal(r.validity, r0.validity, err_msg=what)
    for k in COUNTERS:
        assert c1[k] == c0[k], (what, k)
    for c in r0.state_csr:
        assert all(x.tobytes() == y.tobytes() for x, y in zip(r.state_csr[c], r0.state_csr[c])), what
    n_cells = r.n_groups * r.n_buckets
    for (cid, pt), flagged in zip(q.state_aggs(), q.state_periods()):
        check_state_maps(r, cid, exact_state_maps(truth, q, cid, pt, n_cells, **kw), "%s map %d" % (what, cid))
        if flagged:
            check_state_periods(r, cid, exact_state_periods(truth, q, cid, pt, n_cells, **kw), "%s col %d" % (what, cid))
    return r


@pytest.mark.parametrize("kind", ["rle", "jitter", "raw"])
def test_groupings(eng, kind):
    a, d, truth = state_arena(11, jitter=300 if kind == "jitter" else 0, raw_frac=0.5 if kind == "raw" else 0.0)
    pages = eng.upload_pages(a, d)
    try:
        for sid in (0, 5):
            one = np.array([sid], dtype=np.uint32)
            check(eng, pages, truth, grid_query(truth, columns=PERIODS, series_ids=one), "%s one series %d" % (kind, sid))
            qu = grid_query(truth, columns=PERIODS, width=0, series_ids=one,
                            time_ranges=[(T0 + 20 * STEP, T0 + 150 * STEP), (T0 + 300 * STEP, T0 + 900 * STEP)])
            check(eng, pages, truth, qu, "%s unbucketed %d" % (kind, sid))
        r = check(eng, pages, truth, grid_query(truth, columns=PERIODS, group_by_series=True), kind + " by series")
        assert all(r.period_csr[c][0][-1] > 0 for c, _ in FIELDS)
        qt = grid_query(truth, columns=PERIODS, series_ids=np.arange(0, 8, 2, dtype=np.uint32))
        check(eng, pages, truth, qt, kind + " tags", group_ids=np.array([2, 0, 3, 1], dtype=np.uint32))
        edges = np.array([T0 - 10 * STEP, T0 + 77 * STEP, T0 + 200 * STEP, T0 + 555 * STEP, T0 + 2000 * STEP], dtype=np.int64)
        qe = grid_query(truth, columns=PERIODS, width=0, group_by_series=True)
        qe.n_buckets = 4
        check(eng, pages, truth, qe, kind + " edges", edges=edges)
    finally:
        pages.close()


def test_filters_tombstones_host_resident(eng):
    a, d, truth = state_arena(12)
    tombs = cabi.tombstones([(3, 1, T0 + 50 * STEP, T0 + 120 * STEP), (5, 3, T0, T0 + 300 * STEP),
                             (7, None, T0 + 10 * STEP, T0 + 40 * STEP), (None, None, T0 + 600 * STEP, T0 + 610 * STEP)])
    for host, verify in ((False, False), (True, True)):
        pages = eng.upload_pages(a, d, host_resident=host, verify_on_read=verify)
        try:
            pages.set_tombstones(tombs)
            q = grid_query(truth, columns=PERIODS, predicates=[(1, I64, ">", -8)], time_ranges=[(T0 + 5 * STEP, T0 + 800 * STEP)],
                           group_by_series=True)
            check(eng, pages, truth, q, "filters host=%s" % host, tombstones=tombs)
            r = check(eng, pages, truth, grid_query(truth, columns=PERIODS, group_by_series=True, width=0),
                      "tombstones only host=%s" % host, tombstones=tombs)
            assert None in r.state_periods(3)[5][0]  # series 5's column 3 is NULL from its first row on
        finally:
            pages.close()


def test_overlapping_chunk_files(eng):
    a, d, truth, files, _ = two_file_arena(T0, STEP)
    pages = eng.upload_pages(a, d)
    try:
        pages.set_chunk_files(files)
        col = [PushedAggregate(1, I64, ["state_agg"])]
        for kw in (dict(group_by_series=True), dict(group_by_series=True, width=7 * STEP), dict(series_ids=np.array([2], np.uint32))):
            check(eng, pages, truth, grid_query(truth, columns=col, **kw), "overlap %s" % kw, files=files)
    finally:
        pages.close()


def test_null_time_pages(eng):
    rng = np.random.default_rng(19)
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
        check(eng, pages, truth, grid_query(truth, columns=PERIODS, group_by_series=True), "NULL-time pages")
    finally:
        pages.close()


def test_u64_states_above_2_63_state_at_duration_in(eng):
    b = datagen.ArenaBuilder()
    ts = T0 + np.arange(7, dtype=np.int64) * STEP
    u = np.array([2**64 - 1, 2**63, 2**63, 5, 2**64 - 1, 2**64 - 1, 0], dtype=np.uint64)
    i = np.array([-(2**63), 2**63 - 1, -1, -1, 0, 0, -(2**63)], dtype=np.int64)
    valid = np.array([1, 1, 0, 1, 1, 1, 1], dtype=bool)
    b.add_column_group(0, ts, [(1, I64, i, valid, None), (3, U64, u, valid, None)])
    a, d = b.finish()
    truth = {0: [(ts, {1: (i, valid), 3: (u, valid)})]}
    pages = eng.upload_pages(a, d)
    try:
        r = check(eng, pages, truth, grid_query(truth, columns=PERIODS, width=0), "extremes")
        t = lambda k: T0 + k * STEP
        pu = r.state_periods(3)[0][0]
        assert list(pu.items()) == [(None, [(t(2), t(3))]), (5, [(t(3), t(4))]), (2**63, [(t(1), t(2))]),
                                    (2**64 - 1, [(t(0), t(1)), (t(4), t(6))])]  # (the last point's state 0: no period)
        mu = r.state_maps(3)[0][0]
        assert state_at(pu, t(5), mu) == 2**64 - 1 and state_at(pu, t(6), mu) is None and state_at(pu, t(2), mu) is None
        assert duration_in(mu, 2**64 - 1, t(0) + 1, t(5), pu) == 2 * STEP - 1
        assert duration_in(mu, 2**64 - 1, t(0) + 1, None, pu) == 3 * STEP - 1 and duration_in(mu, 0, t(0), None, pu) == 0
        pi = r.state_periods(1)[0][0]
        assert list(pi) == [None, -(2**63), -1, 0, 2**63 - 1]
        assert pi[-1] == [(t(3), t(4))] and pi[0] == [(t(4), t(6))]
    finally:
        pages.close()


def test_prepared_replay_is_byte_identical(eng):
    a, d, truth = state_arena(16)
    pages = eng.upload_pages(a, d)
    try:
        q = grid_query(truth, columns=PERIODS, group_by_series=True, width=7 * STEP)
        s = eng.prepare(pages, q)
        try:
            off, states, valid, starts, ends = s.state_periods(0)  # before the first run: empty lists
            assert not off.any() and states.size == valid.size == starts.size == ends.size == 0
            s.run()
            first = s.finalize()
            csr = [s.state_periods(k) for k in range(2)]
            n = sum(int(c[0][-1]) for c in csr)
            assert n > 0
            for _ in range(3):
                s.enqueue()
                s.sync()
                r = s.finalize()
                np.testing.assert_array_equal(r.values, first.values)
                for k in range(2):
                    for x, y in zip(s.state_periods(k), csr[k]):
                        assert x.dtype == y.dtype and x.tobytes() == y.tobytes()
            n_cells = first.n_groups * first.n_buckets
            for (cid, pt) in q.state_aggs():
                check_state_periods(first, cid, exact_state_periods(truth, q, cid, pt, n_cells), "prepared %d" % cid)
        finally:
            s.close()
    finally:
        pages.close()


def test_caller_bounds_without_time_span(eng):
    """Caller time bounds that give groups with rows min > max: the start time sort reads all 64 bits."""
    a, d, truth = state_arena(18, n_points=400)
    bounds = np.array([(int(ts[0]), int(ts[-1])) for sid in truth for ts, _ in truth[sid]], dtype=np.int64)
    bounds[::2] = (1, 0)
    pages = eng.upload_pages(a, d)
    try:
        pages.set_time_bounds(bounds)
        check(eng, pages, truth, grid_query(truth, columns=PERIODS, group_by_series=True, width=3 * STEP), "caller bounds")
    finally:
        pages.close()


def test_flagged_and_unflagged_operands(eng):
    """A state_agg and a compact_state_agg in one query, with other aggregates: only the flagged one has periods; a column
    asked for both shares one operand."""
    a, d, truth = state_arena(13)
    pages = eng.upload_pages(a, d)
    try:
        cols = [PushedAggregate(1, I64, ["count", "sum", "median", "gauge_agg", "state_agg", "compact_state_agg"]),
                PushedAggregate(3, U64, ["count", "compact_state_agg"])]
        q = grid_query(truth, columns=cols, group_by_series=True)
        assert q.state_aggs() == [(1, I64), (3, U64)] and q.state_periods() == [True, False]
        r = check(eng, pages, truth, q, "mixed")
        assert set(r.period_csr) == {1}
        s = eng.prepare(pages, q)
        try:
            s.run()
            with pytest.raises(TskvError) as e:
                s.state_periods(1)
            assert e.value.status == cabi.TSKV_ERR_INVALID_ARG
            with pytest.raises(TskvError) as e:
                s.state_periods(2)
            assert e.value.status == cabi.TSKV_ERR_INVALID_ARG
        finally:
            s.close()
    finally:
        pages.close()


def test_one_row_and_equal_time_cells(eng):
    """A cell of one row has a map entry and no period: the reference's compact-agg error. Rows of a series that share one
    time (a page set without chunk files whose column groups overlap) make periods of length 0, which the scan drops: a
    cell whose rows all share one time also answers with that error, where the reference answers NULL / 0."""
    b = datagen.ArenaBuilder()
    b.add_column_group(0, np.array([T0, T0 + 5 * STEP, T0 + 9 * STEP], np.int64), [(1, I64, np.array([4, 5, 4], np.int64), None, None)])
    b.add_column_group(0, np.array([T0 + 20 * STEP], np.int64), [(1, I64, np.array([7], np.int64), None, None)])
    b.add_column_group(0, np.array([T0 + 20 * STEP], np.int64), [(1, I64, np.array([8], np.int64), None, None)])
    a, d = b.finish()
    pages = eng.upload_pages(a, d)
    try:
        q = QueryOption([PushedAggregate(1, I64, ["state_agg"])], width=10 * STEP, first_bucket_start=T0, n_buckets=3)
        r = eng.scan_aggregate(pages, q)
        maps, periods = r.state_maps(1)[0], r.state_periods(1)[0]
        assert maps[0] == {4: 5 * STEP, 5: 4 * STEP}
        assert periods[0] == {4: [(T0, T0 + 5 * STEP)], 5: [(T0 + 5 * STEP, T0 + 9 * STEP)]}
        assert maps[1] == {} and periods[1] == {}
        assert maps[2] == {7: 0, 8: 0} and periods[2] == {}
        assert state_at(periods[1], T0 + 15 * STEP, maps[1]) is None
        with pytest.raises(CompactAggError):
            state_at(periods[2], T0 + 20 * STEP, maps[2])
        with pytest.raises(CompactAggError):
            duration_in(maps[2], 7, T0, None, periods[2])
        assert duration_in(maps[2], 7) == 0  # (without a start time the map answers)
    finally:
        pages.close()


def test_refusals(eng):
    a, d, truth = state_arena(15, n_series=4, n_points=50)
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
        one = dict(series_ids=np.array([1], np.uint32))
        op = lambda cid=1, pt=I64: PushedAggregate(cid, pt, ["state_agg"])
        flag = lambda c: setattr(c, "agg_mask", cabi.TSKV_STATE_PERIODS)
        raw = lambda cols, **kw: _RawQuery(cols, first_bucket_start=0, n_buckets=1, **dict(one, **kw))
        assert prepare_status(raw([op()])) == cabi.TSKV_OK
        # other masks on a state agg operand
        for m in (cabi.TSKV_AGG_COUNT, cabi.TSKV_STATE_PERIODS | cabi.TSKV_AGG_COUNT, 0x40):
            assert prepare_status(raw([op()], patch=lambda c, m=m: setattr(c, "agg_mask", m))) == INV
        # the flag on every other operand kind
        for kind in ("median", "increase", "mode", "count_distinct", "gauge_agg"):
            assert prepare_status(raw([PushedAggregate(1, I64, [kind])], patch=flag)) == INV, kind
        pair = QueryOption([], pairs=[(1, I64, 3, U64)], first_bucket_start=0, n_buckets=1, **one)
        cq = pair.to_c()
        cq.columns[0].agg_mask = cabi.TSKV_STATE_PERIODS
        h = C.c_void_p()
        assert eng.lib.tskvgpu_scan_prepare(eng.ctx, pages.handle, C.byref(cq), C.byref(h)) == INV
        # every state agg refusal applies with the flag set
        assert status(grid_query(truth, columns=[op(2, F64)], **one)) == INV
        assert status(grid_query(truth, columns=[op(5, cabi.TSKV_PT_BOOL)], **one)) == INV
        assert status(grid_query(truth, columns=[op(0, cabi.TSKV_PT_TIME)], **one)) == INV
        assert status(grid_query(truth, columns=[PushedAggregate(1, I64, ["count"]), op(1, U64)], **one)) == INV
        many = lambda n: [PushedAggregate(100 + i, I64, ["count"]) for i in range(n)] + [op()] * 7
        assert status(grid_query(truth, columns=many(119), **one)) == cabi.TSKV_OK
        assert status(grid_query(truth, columns=many(120), **one)) == INV
        assert status(grid_query(truth, columns=[op()])) == UNS
        assert status(grid_query(truth, columns=[op()], series_ids=np.array([0, 1], np.uint32)),
                      group_ids=np.array([0, 0], np.uint32), n_groups=1) == UNS
        assert status(grid_query(truth, columns=[op()], group_by_series=True), slide=W // 5) == UNS
        edges = np.array([T0 - 10 * STEP, T0 + 77 * STEP, T0 + 200 * STEP], dtype=np.int64)
        ql = grid_query(truth, columns=[op()], width=0, group_by_series=True)
        ql.n_buckets = 1
        assert status(ql, edges=edges, labels=np.array([0, 0], np.uint32)) == UNS
        assert prepare_status(raw([op()], flags=cabi.TSKV_QUERY_MULTI_RANK)) == UNS
        b = datagen.ArenaBuilder()
        b.add_column_group(0, np.array([-(2**62) * 2, 2**62, 2**63 - 1], dtype=np.int64),
                           [(1, I64, np.array([1, 2, 3], dtype=np.int64), None, datagen.encode_raw)])
        wa, wd = b.finish()
        wide = eng.upload_pages(wa, wd)
        try:
            with pytest.raises(TskvError) as e:
                eng.scan_aggregate(wide, QueryOption([op()], n_buckets=1))
            assert e.value.status == UNS
            r = eng.scan_aggregate(wide, QueryOption([op()], n_buckets=1, time_ranges=[(0, 2**63 - 1)]))
            assert r.state_periods(1)[0][0] == {2: [(2**62, 2**63 - 1)]}
        finally:
            wide.close()
        b = datagen.ArenaBuilder()
        b.add_column_group(0, T0 + np.arange(4, dtype=np.int64) * STEP, [(1, I64, np.arange(4, dtype=np.int64), None, None)])
        b.add_column_group(0, T0 + np.arange(10, 14, dtype=np.int64) * STEP, [(3, U64, np.arange(4, dtype=np.uint64), None, None)])
        ma, md = b.finish()
        missing = eng.upload_pages(ma, md)
        try:
            with pytest.raises(TskvError) as e:
                eng.scan_aggregate(missing, QueryOption([op()], n_buckets=1))
            assert e.value.status == UNS
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
                s.state_periods(1)
            assert e.value.status == INV
        finally:
            s.close()
    finally:
        pages.close()
