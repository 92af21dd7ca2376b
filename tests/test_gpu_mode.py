"""mode(x) and COUNT(DISTINCT x) (TSKV_QUERY_N_MODES / _N_DISTINCTS) through the scan against tests/mode_reference.py, bit
for bit: RLE, jittered and raw time pages with NULLs; bucketed, GROUP BY series, unbucketed, tag-group, edge and label
grids; predicates, tombstones, host-resident pages with CRC on read; overlapping chunk files; ties, one-value and
all-NULL cells and f64 specials; GROUP BY series over more cells than medians allow; a query mixing every other
operand kind; repeated run / enqueue; every refusal."""
import ctypes as C

import numpy as np
import pytest

from cnosdb_b200 import cabi, datagen
from cnosdb_b200.engine import Engine, PushedAggregate, QueryOption, TskvError
from tests.exact_arenas import two_file_arena
from tests.helpers import bucket_spec, random_arena
from tests.mode_reference import check_distinct, check_mode, exact_mode_cells

pytestmark = pytest.mark.gpu

I64, U64, F64 = cabi.TSKV_PT_I64, cabi.TSKV_PT_U64, cabi.TSKV_PT_F64
T0, STEP, W = 1_000_000, 1000, 50_000
FIELDS = ((1, I64), (2, F64), (3, U64))
BOTH = [PushedAggregate(c, pt, ["mode", "count_distinct"]) for c, pt in FIELDS]


@pytest.fixture(scope="module")
def eng():
    e = Engine(0)
    yield e
    e.close()


def arena(seed, null_frac=0.2, jitter=0, raw_frac=0.0, n_series=24, n_points=400, fields=FIELDS):
    rng = np.random.default_rng(seed)
    return random_arena(rng, n_series=n_series, n_points=n_points, fields=fields, null_frac=null_frac, t0=T0, step=STEP,
                        jitter=jitter, raw_frac=raw_frac, multi_cg=True)


def grid_query(truth, columns=BOTH, **kw):
    t_hi = max(int(ts[-1]) for cgs in truth.values() for ts, _ in cgs if len(ts))
    kw.setdefault("width", W)
    fbs, nb = bucket_spec(T0 - 10 * STEP, t_hi + STEP, kw["width"]) if kw["width"] > 0 else (0, 1)
    return QueryOption(list(columns), first_bucket_start=fbs, n_buckets=nb, **kw)


def check_modes(res, truth, q, what, **kw):
    """Every mode and distinct output of res (they come last: the modes in column order, then the distincts)."""
    n_cells = res.n_groups * res.n_buckets
    modes = [c for c in q.columns if c.mode]
    dists = [c for c in q.columns if c.count_distinct]
    j0 = len(res.names) - len(modes) - len(dists)
    cache = {}
    for k, c in enumerate(modes + dists):
        key = (c.column_id, c.phys_type)
        if key not in cache:
            cache[key] = exact_mode_cells(truth, q, c.column_id, c.phys_type, n_cells, **kw)
        if k < len(modes):
            check_mode(res, j0 + k, cache[key], what="%s mode %d" % (what, k))
        else:
            check_distinct(res, j0 + k, cache[key], what="%s distinct %d" % (what, k))
    assert any(e[1].any() for e in cache.values()), what


@pytest.mark.parametrize("kind", ["rle", "jitter", "raw"])
def test_groupings(eng, kind):
    a, d, truth = arena(1, jitter=300 if kind == "jitter" else 0, raw_frac=0.5 if kind == "raw" else 0.0)
    pages = eng.upload_pages(a, d)
    try:
        sel = np.arange(0, 24, 2, dtype=np.uint32)
        q = grid_query(truth, series_ids=sel)
        check_modes(eng.scan_aggregate(pages, q), truth, q, kind + " bucket")
        qs = grid_query(truth, series_ids=sel, group_by_series=True)
        check_modes(eng.scan_aggregate(pages, qs), truth, qs, kind + " series")
        qu = grid_query(truth, width=0, time_ranges=[(T0 + 20 * STEP, T0 + 150 * STEP), (T0 + 300 * STEP, T0 + 900 * STEP)])
        check_modes(eng.scan_aggregate(pages, qu), truth, qu, kind + " unbucketed, two ranges")
        gids = (sel % 3).astype(np.uint32)
        check_modes(eng.scan_aggregate(pages, q, group_ids=gids, n_groups=3), truth, q, kind + " tags", group_ids=gids)
        edges = np.array([T0 - 10 * STEP, T0 + 77 * STEP, T0 + 200 * STEP, T0 + 555 * STEP, T0 + 2000 * STEP], dtype=np.int64)
        qe = grid_query(truth, width=0, series_ids=sel)
        qe.n_buckets = 4
        check_modes(eng.scan_aggregate(pages, qe, edges=edges), truth, qe, kind + " edges", edges=edges)
        labels = np.array([1, 0, 1, 0], dtype=np.uint32)
        ql = grid_query(truth, width=0, series_ids=sel)
        ql.n_buckets = 2
        check_modes(eng.scan_aggregate(pages, ql, edges=edges, labels=labels), truth, ql, kind + " labels", edges=edges,
                    labels=labels)
    finally:
        pages.close()


SPECIALS = np.array([0x0000000000000000, 0x8000000000000000, 0x7FF8000000000000, 0x7FF8000000000001, 0xFFF8000000000000,
                     0x7FF0000000000000, 0xFFF0000000000000, 0x3FF0000000000000], dtype=np.uint64).view(np.float64)
POOLS = {I64: np.array([-3, 0, 7, -(2**63), 2**63 - 1], dtype=np.int64), U64: np.array([0, 5, 2**63, 2**64 - 1], dtype=np.uint64),
         F64: SPECIALS}


def pool_arena(seed, n_series=16, n_points=300, null_frac=0.3):
    """Values drawn from a few per column (integer extremes, f64 -0.0 / +0.0, NaN payloads, infinities): repeated
    values, ties, one-value cells; every 7th series' column group is all NULL in column 3."""
    rng = np.random.default_rng(seed)
    b = datagen.ArenaBuilder()
    truth = {}
    for sid in range(n_series):
        t_start = T0
        for _ in range(1 + int(rng.random() < 0.3)):
            n = int(rng.integers(1, n_points + 1))
            ts = t_start + np.arange(n, dtype=np.int64) * STEP
            t_start = int(ts[-1]) + STEP
            fl, cols = [], {}
            for col, pt in FIELDS:
                pool = POOLS[pt][: int(rng.integers(1, len(POOLS[pt]) + 1))]
                vals = pool[rng.integers(0, len(pool), n)]
                valid = rng.random(n) >= null_frac
                if col == 3 and sid % 7 == 0:
                    valid[:] = False
                fl.append((col, pt, vals, valid, datagen.encode_raw if rng.random() < 0.3 else None))
                cols[col] = (vals, valid)
            b.add_column_group(sid, ts, fl)
            truth.setdefault(sid, []).append((ts, cols))
    arena_, descs = b.finish()
    return arena_, descs, truth


def test_ties_specials_and_empty_cells(eng):
    a, d, truth = pool_arena(11)
    pages = eng.upload_pages(a, d)
    try:
        for kw in (dict(group_by_series=True), dict(), dict(width=0), dict(width=STEP, group_by_series=True)):
            q = grid_query(truth, **kw)
            check_modes(eng.scan_aggregate(pages, q), truth, q, "pools %s" % kw)
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
            check_modes(eng.scan_aggregate(pages, q), truth, q, "filters host=%s" % host, tombstones=tombs)
        finally:
            pages.close()


def test_overlapping_chunk_files(eng):
    """Two overlapping chunk files per series: the merged rows are gathered too."""
    a, d, truth, files, _ = two_file_arena(T0, STEP)
    pages = eng.upload_pages(a, d)
    try:
        pages.set_chunk_files(files)
        for gbs in (True, False):
            q = grid_query(truth, columns=BOTH[:2], group_by_series=gbs)
            check_modes(eng.scan_aggregate(pages, q), truth, q, "overlap gbs=%s" % gbs, files=files)
    finally:
        pages.close()


def test_more_cells_than_medians_allow(eng):
    """GROUP BY series with 1-ns-wide buckets: more than TSKV_MAX_MEDIAN_CELLS cells, memory in proportion to the rows."""
    a, d, truth = pool_arena(12, n_series=24, n_points=400)
    pages = eng.upload_pages(a, d)
    try:
        q = grid_query(truth, columns=[PushedAggregate(1, I64, ["mode", "count_distinct"])], width=2, group_by_series=True)
        res = eng.scan_aggregate(pages, q)
        assert res.n_groups * res.n_buckets > cabi.TSKV_MAX_MEDIAN_CELLS
        check_modes(res, truth, q, "many cells")
    finally:
        pages.close()


def test_mixed_query_outputs_and_counters(eng):
    """One query grouped by series with projected aggregates, a pair, a median, an increase, modes and distincts on the
    same and on different columns: the other outputs equal those of the query without modes and distincts, and the
    reader counters equal those of that query with the unprojected operands added as COUNT columns."""
    a, d, truth = arena(3)
    pages = eng.upload_pages(a, d)
    try:
        base = [PushedAggregate(1, I64, ["count", "sum", "min", "max", "median"]), PushedAggregate(2, F64, ["count", "increase"])]
        extra = [PushedAggregate(1, I64, ["mode"]), PushedAggregate(2, F64, ["mode", "count_distinct"]),
                 PushedAggregate(3, U64, ["count_distinct"]), PushedAggregate(1, I64, ["count_distinct", "mode"])]
        kw = dict(pairs=[(1, I64, 2, F64)], predicates=[(3, U64, ">=", 0)], group_by_series=True)
        q = grid_query(truth, columns=base + extra, **kw)
        r = eng.scan_aggregate(pages, q)
        c = eng.counters()
        q0 = grid_query(truth, columns=base, **kw)
        r0 = eng.scan_aggregate(pages, q0)
        names0 = q0.output_names()
        for j0, name in enumerate(names0):
            j = r.names.index(name)
            np.testing.assert_array_equal(r.validity[j], r0.validity[j0], err_msg=str(name))
            ok = r.validity[j]
            x, y = r.values[j][ok], r0.values[j0][ok]
            if name[1] in ("c", "m2x", "m2y", "increase") or (name[1] in ("sum", "mean") and r.phys.get(name[0]) == F64):
                np.testing.assert_allclose(x.view(np.float64), y.view(np.float64), rtol=1e-12, atol=1e-300, err_msg=str(name))
            else:
                np.testing.assert_array_equal(x, y, err_msg=str(name))
        assert r.names[len(names0):] == [(1, "mode"), (2, "mode"), (1, "mode"), (2, "count_distinct"), (3, "count_distinct"),
                                         (1, "count_distinct")]
        check_modes(r, truth, q, "mixed")
        # the operand of column 3 is not projected: the counters match the query with it as a COUNT column
        qc = grid_query(truth, columns=base + [PushedAggregate(3, U64, ["count"])], **kw)
        eng.scan_aggregate(pages, qc)
        cc = eng.counters()
        for k in ("page_read_count", "page_read_bytes", "points_decoded", "rows_in_range", "pruned_page_count"):
            assert c[k] == cc[k], k
    finally:
        pages.close()


def test_repeated_run_and_enqueue(eng):
    """run() and the captured enqueue() replays give identical outputs (the slices, cursors and run results are reset
    on every pass)."""
    a, d, truth = arena(6)
    q = grid_query(truth, group_by_series=True)
    pages = eng.upload_pages(a, d)
    try:
        s = eng.prepare(pages, q)
        try:
            s.run()
            first = s.finalize()
            check_modes(first, truth, q, "run")
            for _ in range(3):
                s.enqueue()
                s.sync()
                r = s.finalize()
                for j in range(len(first.names)):
                    np.testing.assert_array_equal(r.values[j], first.values[j])
                    np.testing.assert_array_equal(r.validity[j], first.validity[j])
        finally:
            s.close()
    finally:
        pages.close()


class _RawQuery(QueryOption):
    """A query whose last operand entry is rewritten by `patch`, with extra flag bits."""

    def __init__(self, *a, patch=None, flags=0, **kw):
        super().__init__(*a, **kw)
        self.patch, self.flags = patch, flags

    def to_c(self):
        q = super().to_c()
        n = len(self.projected()) + cabi.query_n_modes(q.reserved) + cabi.query_n_distincts(q.reserved) - 1
        if self.patch:
            self.patch(q.columns[n])
        q.reserved |= self.flags
        return q


@pytest.mark.parametrize("agg", ["mode", "count_distinct"])
def test_refusals(eng, agg):
    a, d, truth = arena(5, n_series=4, n_points=50)
    pages = eng.upload_pages(a, d)
    try:
        def status(q, **kw):
            try:
                eng.scan_aggregate(pages, q, **kw)
            except TskvError as e:
                return e.status
            return cabi.TSKV_OK

        def prepare_status(q, slide=None):
            h = C.c_void_p()
            cq = q.to_c()
            st = (eng.lib.tskvgpu_scan_prepare_sliding(eng.ctx, pages.handle, C.byref(cq), slide, C.byref(h)) if slide
                  else eng.lib.tskvgpu_scan_prepare(eng.ctx, pages.handle, C.byref(cq), C.byref(h)))
            assert not h.value or st == cabi.TSKV_OK
            if h.value:
                eng.lib.tskvgpu_scan_destroy(eng.ctx, h)
            return st
        INV, UNS = cabi.TSKV_ERR_INVALID_ARG, cabi.TSKV_ERR_UNSUPPORTED
        op = lambda cid=1, pt=I64: PushedAggregate(cid, pt, [agg])
        assert status(grid_query(truth, columns=[op()] * 8)) == cabi.TSKV_OK
        assert status(grid_query(truth, columns=[op()] * 9)) == INV
        assert status(grid_query(truth, columns=[op(5, cabi.TSKV_PT_BOOL)])) == INV
        assert status(grid_query(truth, columns=[op(0, cabi.TSKV_PT_TIME)])) == INV
        assert status(grid_query(truth, columns=[op(1, 9)])) == INV
        assert status(grid_query(truth, columns=[PushedAggregate(1, I64, ["count"]), op(1, F64)])) == INV
        assert status(grid_query(truth, columns=[op(1, I64), op(1, U64)])) == INV
        many = lambda n: [PushedAggregate(100 + i, I64, ["count"]) for i in range(n)] + [op()] * 8
        assert status(grid_query(truth, columns=many(118))) == cabi.TSKV_OK  # 126 columns
        assert status(grid_query(truth, columns=many(119))) == INV
        masked = _RawQuery([op()], first_bucket_start=0, n_buckets=1, patch=lambda c: setattr(c, "agg_mask", cabi.TSKV_AGG_COUNT))
        assert prepare_status(masked) == INV
        with pytest.raises(ValueError):
            eng.scan_aggregate(pages, grid_query(truth, columns=[op()]), slide=W // 5)
        assert prepare_status(grid_query(truth, columns=[op()]), slide=W // 5) == UNS
        with pytest.raises(ValueError):
            eng.scan_aggregate(pages, grid_query(truth, columns=[op()], multi_rank=True, series_ids=np.arange(4, dtype=np.uint32)))
        mr = _RawQuery([op()], first_bucket_start=0, n_buckets=1, flags=cabi.TSKV_QUERY_MULTI_RANK)
        assert prepare_status(mr) == UNS
        # gathers x cells of 2^31 or more: GROUP BY tags into 2^31 groups (refused before anything is allocated)
        gids = np.arange(4, dtype=np.uint32)
        assert status(QueryOption([op()], n_buckets=1), group_ids=gids, n_groups=1 << 31) == UNS
        s = eng.prepare(pages, grid_query(truth, columns=[op()]))
        try:
            s.run()
            for call in (s.partials, s.exchange_view, s.exchange, lambda: s.merge_gathered(1, 1)):
                with pytest.raises(TskvError) as e:
                    call()
                assert e.value.status == UNS
        finally:
            s.close()
    finally:
        pages.close()
