"""Counter increases (TSKV_QUERY_N_INCREASES) through the scan against tests/increase_reference.py: integers bit for bit,
f64 within the SUM rules. Every grouping a cell of one series allows (GROUP BY series, tag groups of one series each,
explicit edges, the unbucketed scan of one series) over RLE, jittered and raw time pages with several column groups per
series written out of time order; simple8b, gorilla and raw values; buckets straddling pages; empty, all-NULL and
filtered pages inside a chain; time-range gaps; predicates, tombstones, NULL-time pages, host-resident pages with CRC on read; merge groups at the
start, middle and end of a series; every refusal; 1 / 3 / 4 / 8 ranks, with chunk files, tombstones and unselected
series, and one series split over ranks by time; random queries scanned twice; the reference's increase.slt answers."""
import ctypes as C

import numpy as np
import pytest

from cnosdb_b200 import cabi, datagen
from cnosdb_b200.engine import Engine, PushedAggregate, QueryOption, TskvError
from tests.helpers import bucket_spec, random_arena
from tests.increase_reference import check_increase, exact_increase_cells, load_golden
from tests.ranks import RankScans, layouts, multi_rank
from tests.test_increase_reference import golden_tb2

pytestmark = pytest.mark.gpu

I64, U64, F64 = cabi.TSKV_PT_I64, cabi.TSKV_PT_U64, cabi.TSKV_PT_F64
T0, STEP, W = 1_000_000, 1000, 50_000
FIELDS = ((1, I64), (2, F64), (3, U64))
INCS = [PushedAggregate(c, pt, ["increase"]) for c, pt in FIELDS]
DT = {I64: np.int64, U64: np.uint64, F64: np.float64}


@pytest.fixture(scope="module")
def eng():
    e = Engine(0)
    yield e
    e.close()


def arena(seed, null_frac=0.2, jitter=0, raw_frac=0.0, n_series=12, n_points=400):
    rng = np.random.default_rng(seed)
    return random_arena(rng, n_series=n_series, n_points=n_points, fields=FIELDS, null_frac=null_frac, t0=T0, step=STEP,
                        jitter=jitter, raw_frac=raw_frac, multi_cg=True)


def t_hi(truth):
    return max(int(ts[-1]) for cgs in truth.values() for ts, _ in cgs if len(ts))


def grid_query(truth, columns=INCS, **kw):
    w = kw.setdefault("width", W)
    fbs, nb = bucket_spec(T0 - 10 * STEP, t_hi(truth) + STEP, w) if w > 0 else (0, 1)
    return QueryOption(list(columns), first_bucket_start=fbs, n_buckets=nb, **kw)


def check_increases(res, truth, q, what, min_valid=1, **kw):
    n_cells = res.n_groups * res.n_buckets
    incs = [c for c in q.columns if c.increase]
    assert incs
    for k, c in enumerate(incs):
        exact = exact_increase_cells(truth, q, c.column_id, c.phys_type, n_cells, **kw)
        j = len(res.names) - len(incs) + k  # (the increase outputs come last, in column order)
        check_increase(res, j, exact, c.phys_type, what="%s increase %d" % (what, k))
        assert exact[1].sum() >= min_valid, what


def scan_all_groupings(eng, pages, truth, what, **kw):
    sel = np.array(sorted(truth)[::2], dtype=np.uint32)
    qs = grid_query(truth, series_ids=sel, group_by_series=True, **kw)
    check_increases(eng.scan_aggregate(pages, qs), truth, qs, what + " series")
    qa = grid_query(truth, group_by_series=True, **kw)
    check_increases(eng.scan_aggregate(pages, qa), truth, qa, what + " every series")
    q = grid_query(truth, series_ids=sel, **kw)
    gids = np.random.default_rng(len(sel)).permutation(len(sel)).astype(np.uint32)  # one series per group, shuffled
    check_increases(eng.scan_aggregate(pages, q, group_ids=gids, n_groups=len(sel) + 2), truth, q, what + " tags",
                    group_ids=gids)
    one = sel[1:2]
    qu = grid_query(truth, width=0, series_ids=one,
                    time_ranges=[(T0 + 20 * STEP, T0 + 150 * STEP), (T0 + 300 * STEP, T0 + 900 * STEP)], **kw)
    check_increases(eng.scan_aggregate(pages, qu), truth, qu, what + " unbucketed one series, two ranges")
    qb = grid_query(truth, series_ids=one, **kw)
    check_increases(eng.scan_aggregate(pages, qb), truth, qb, what + " buckets of one series")
    edges = np.array([T0 - 10 * STEP, T0 + 77 * STEP, T0 + 200 * STEP, T0 + 333 * STEP, max(t_hi(truth), T0 + 555 * STEP) + STEP],
                     dtype=np.int64)
    qe = grid_query(truth, width=0, series_ids=sel, group_by_series=True, **kw)
    qe.n_buckets = 4
    check_increases(eng.scan_aggregate(pages, qe, edges=edges), truth, qe, what + " edges", edges=edges)


@pytest.mark.parametrize("kind", ["rle", "jitter", "raw"])
def test_groupings(eng, kind):
    a, d, truth = arena(1, jitter=300 if kind == "jitter" else 0, raw_frac=0.5 if kind == "raw" else 0.0)
    pages = eng.upload_pages(a, d)
    try:
        scan_all_groupings(eng, pages, truth, kind)
    finally:
        pages.close()


def chain_arena(seed, encoders):
    """Four series, each a chain of column groups added in reverse time order (descriptor order != time order) whose
    pages are cut at 37-row steps so that buckets straddle them; inside the chain an empty-operand page (operand
    absent), an all-NULL page, and pages of every value encoder in `encoders` (one per series)."""
    rng = np.random.default_rng(seed)
    b = datagen.ArenaBuilder()
    truth = {}
    for sid, enc in enumerate(encoders):
        cgs = []
        t = T0 + sid * 7
        for k in range(8):
            n = 37 + int(rng.integers(0, 60))
            ts = t + np.arange(n, dtype=np.int64) * STEP
            t = int(ts[-1]) + STEP * (1 + int(rng.integers(0, 3)))
            fields, cols = [], {}
            for cid, pt in FIELDS:
                if k == 2 and cid == 1:
                    continue  # the column group has no page of column 1
                v = np.cumsum(rng.integers(-2, 6, n)).astype(DT[pt]) if pt != U64 else \
                    np.cumsum(rng.integers(0, 6, n)).astype(np.uint64)
                if pt == F64:
                    v = v + rng.random(n)
                valid = np.zeros(n, dtype=bool) if k == 4 else rng.random(n) > 0.15
                fields.append((cid, pt, v, valid, enc(pt)))
                cols[cid] = (v, valid)
            cgs.append((ts, fields, cols))
        for ts, fields, _ in reversed(cgs):
            b.add_column_group(sid, ts, [f if f[4] is not None else f[:4] for f in fields])
        truth[sid] = [(ts, cols) for ts, _, cols in cgs]
    a, d = b.finish()
    return a, d, truth


def test_chains_every_value_encoder(eng):
    """Value encoders per series (the defaults: simple8b integers and gorilla floats; raw integers); RLE time pages come
    from regular steps, and the per-series offsets make buckets straddle pages."""
    encs = [lambda pt: None,
            lambda pt: datagen.encode_floats if pt == F64 else None,
            lambda pt: datagen.encode_raw if pt != F64 else None,
            lambda pt: None]
    a, d, truth = chain_arena(3, encs)
    pages = eng.upload_pages(a, d)
    try:
        for w in (W, 3 * STEP, 1_000 * STEP):
            qs = grid_query(truth, group_by_series=True, width=w)
            check_increases(eng.scan_aggregate(pages, qs), truth, qs, "chains w=%d" % w)
        # fully filtered and pruned pages in the middle of a chain: a predicate and a time-range gap
        qf = grid_query(truth, group_by_series=True, predicates=[(2, F64, "<", 40.0)],
                        time_ranges=[(T0, T0 + 150 * STEP), (T0 + 260 * STEP, T0 + 2000 * STEP)])
        check_increases(eng.scan_aggregate(pages, qf), truth, qf, "chains filtered")
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
            check_increases(eng.scan_aggregate(pages, q), truth, q, "filters host=%s" % host, tombstones=tombs)
        finally:
            pages.close()


def test_null_time_pages(eng):
    """Raw time pages that mark rows NULL: those rows are not selected (the reference marks their operand values
    NULL)."""
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
                v = np.cumsum(rng.integers(-1, 5, n)).astype(DT[pt]) if pt != U64 else np.cumsum(rng.integers(0, 5, n)).astype(np.uint64)
                valid = rng.random(n) > 0.1
                fields.append((cid, pt, v, valid))
                cols[cid] = (v, valid & tvalid)
            b.add_page(datagen.build_page(datagen.encode_raw(ts[tvalid]), n, tvalid), sid, 0, cabi.TSKV_PT_TIME, n)
            for cid, pt, v, valid in fields:
                kept = v[valid].view(np.int64) if pt == U64 else v[valid]
                enc = datagen.encode_floats if pt == F64 else datagen.encode_integers
                b.add_page(datagen.build_page(enc(kept), n, valid), sid, cid, pt, n)
            cgs.append((ts, cols))
        truth[sid] = cgs
    a, d = b.finish()
    pages = eng.upload_pages(a, d)
    try:
        q = grid_query(truth, group_by_series=True)
        check_increases(eng.scan_aggregate(pages, q), truth, q, "NULL-time pages")
    finally:
        pages.close()


def merge_arena(seed):
    """Three series whose chains hold a merge group (two overlapping chunk files) at the start, in the middle and at the
    end: -> (arena, descs, truth, files)."""
    rng = np.random.default_rng(seed)
    b = datagen.ArenaBuilder()
    truth, files = {}, []
    spans = {0: [(0, 120, 1), (60, 200, 2), (200, 320, 1), (330, 450, 1)],
             1: [(0, 100, 1), (110, 230, 1), (180, 300, 2), (310, 420, 1)],
             2: [(0, 100, 1), (110, 230, 1), (250, 380, 1), (300, 420, 2)]}
    for sid, chain in spans.items():
        cgs = []
        for lo, hi, f in reversed(chain):  # (descriptor order != time order)
            n = hi - lo
            ts = T0 + np.arange(lo, hi, dtype=np.int64) * STEP
            fields, cols = [], {}
            for cid, pt in FIELDS:
                v = np.cumsum(rng.integers(-2, 6, n)).astype(DT[pt]) if pt != U64 else np.cumsum(rng.integers(0, 6, n)).astype(np.uint64)
                valid = rng.random(n) > 0.2
                fields.append((cid, pt, v, valid))
                cols[cid] = (v, valid)
            b.add_column_group(sid, ts, fields)
            files.append(f)
            cgs.append((ts, cols))
        truth[sid] = cgs
    a, d = b.finish()
    return a, d, truth, np.asarray(files, dtype=np.uint64)


def test_merge_groups_start_middle_end(eng):
    a, d, truth, files = merge_arena(4)
    pages = eng.upload_pages(a, d)
    try:
        pages.set_chunk_files(files)
        for w in (W, 7 * STEP):
            q = grid_query(truth, group_by_series=True, width=w)
            check_increases(eng.scan_aggregate(pages, q), truth, q, "merge w=%d" % w, files=files)
        qu = grid_query(truth, width=0, series_ids=np.array([1], dtype=np.uint32))
        check_increases(eng.scan_aggregate(pages, qu), truth, qu, "merge unbucketed", files=files)
        qp = grid_query(truth, group_by_series=True, predicates=[(3, U64, ">", 20)])
        check_increases(eng.scan_aggregate(pages, qp), truth, qp, "merge predicate", files=files)
    finally:
        pages.close()


def test_special_values(eng):
    """NaN of both signs, +-inf, -0.0 / +0.0, i64 / u64 wrapping at the extremes, one value, equal runs."""
    b = datagen.ArenaBuilder()
    truth = {}
    nn = float(np.uint64(0xFFF8000000000000).view(np.float64))
    cases = {
        0: (F64, [1.0, np.nan, 2.0]), 1: (F64, [nn, 1.0]), 2: (F64, [1.0, np.inf, 0.5]), 3: (F64, [0.0, -0.0, 0.0]),
        4: (F64, [2.5]), 5: (F64, [3.25] * 6), 6: (I64, [-2**63, 2**63 - 1, 0, 2**63 - 1]), 7: (I64, [2**63 - 1, -2**63]),
        8: (U64, [0, 2**64 - 1, 0, 2**64 - 1]), 9: (U64, [2**63, 1, 2**63]), 10: (I64, [-7] * 5), 11: (F64, [-np.inf, 1.0]),
    }
    for sid, (pt, vals) in cases.items():
        cid = {I64: 1, F64: 2, U64: 3}[pt]
        n = len(vals)
        ts = T0 + np.arange(n, dtype=np.int64) * STEP
        v = np.array(vals, dtype=DT[pt])
        b.add_column_group(sid, ts, [(cid, pt, v, None)])
        truth[sid] = [(ts, {cid: (v, np.ones(n, dtype=bool))})]
    a, d = b.finish()
    pages = eng.upload_pages(a, d)
    try:
        q = grid_query(truth, group_by_series=True, width=0)
        res = eng.scan_aggregate(pages, q)
        check_increases(res, truth, q, "special values")
        v, ok = res.column(1, "increase")
        assert v[6, 0] == 2**63 - 2 and v[7, 0] == -2**63  # (MAX - MIN wraps to -1; 0 resets; MAX - 0)
        u, _ = res.column(3, "increase")
        assert u[8, 0] == 2**64 - 2
        f, _ = res.column(2, "increase")
        assert np.isnan(f[0, 0]) and np.isnan(f[1, 0]) and f[4, 0] == 0.0 and f[5, 0] == 0.0
    finally:
        pages.close()


def test_mixed_query_outputs_and_counters(eng):
    """Projected aggregates, a pair, a median and increases of a projected and of an unprojected column: the other outputs
    equal those of the query without increases; the reader counters equal those of that query with the unprojected
    operand added as a COUNT column; graph replays meet the reference."""
    a, d, truth = arena(3)
    pages = eng.upload_pages(a, d)
    try:
        base = [PushedAggregate(1, I64, ["count", "sum", "mean", "min", "max", "median"]), PushedAggregate(2, F64, ["count", "stddev"])]
        with_inc = [PushedAggregate(1, I64, ["count", "sum", "mean", "min", "max", "median", "increase"]),
                    PushedAggregate(2, F64, ["count", "stddev"]), PushedAggregate(3, U64, ["increase"]),
                    PushedAggregate(2, F64, ["increase"])]
        kw = dict(pairs=[(1, I64, 2, F64)], predicates=[(2, F64, ">=", -1e9)], group_by_series=True)
        q = grid_query(truth, columns=with_inc, **kw)
        r = eng.scan_aggregate(pages, q)
        c = eng.counters()
        q0 = grid_query(truth, columns=base, **kw)
        r0 = eng.scan_aggregate(pages, q0)
        for j0, name in enumerate(q0.output_names()):
            j = r.names.index(name)
            np.testing.assert_array_equal(r.validity[j], r0.validity[j0], err_msg=str(name))
            ok = r.validity[j]
            x, y = r.values[j][ok], r0.values[j0][ok]
            if name[1] in ("m2", "c", "m2x", "m2y") or (name[1] in ("sum", "mean") and r.phys.get(name[0]) == F64):
                np.testing.assert_allclose(x.view(np.float64), y.view(np.float64), rtol=1e-12, atol=1e-300, err_msg=str(name))
            else:
                np.testing.assert_array_equal(x, y, err_msg=str(name))
        assert r.names[-3:] == [(1, "increase"), (3, "increase"), (2, "increase")]
        check_increases(r, truth, q, "mixed")
        qc = grid_query(truth, columns=base + [PushedAggregate(3, U64, ["count"])], **kw)
        eng.scan_aggregate(pages, qc)
        cc = eng.counters()
        for k in ("page_read_count", "page_read_bytes", "points_decoded", "rows_in_range", "pruned_page_count"):
            assert c[k] == cc[k], k
        assert c["kernel_launches"] >= cc["kernel_launches"] + 6
        s = eng.prepare(pages, q)
        try:
            for _ in range(3):
                s.enqueue()
                s.sync()
                check_increases(s.finalize(), truth, q, "graph replay")
        finally:
            s.close()
    finally:
        pages.close()


class _RawQuery(QueryOption):
    """A query whose last increase operand is rewritten by `patch` (engine.QueryOption writes agg_mask 0)."""

    def __init__(self, *a, patch=None, **kw):
        super().__init__(*a, **kw)
        self.patch = patch

    def to_c(self):
        q = super().to_c()
        n = (len(self.projected()) + 2 * len(self.pairs) + cabi.query_n_medians(q.reserved) +
             cabi.query_n_increases(q.reserved) - 1)
        self.patch(q.columns[n])
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

        def prepare_status(q, slide=None):
            h = C.c_void_p()
            cq = q.to_c()
            st = (eng.lib.tskvgpu_scan_prepare_sliding(eng.ctx, pages.handle, C.byref(cq), slide, C.byref(h)) if slide
                  else eng.lib.tskvgpu_scan_prepare(eng.ctx, pages.handle, C.byref(cq), C.byref(h)))
            assert not h.value or st == cabi.TSKV_OK
            if h.value:
                eng.lib.tskvgpu_scan_destroy(eng.ctx, h)
            return st
        INV, UNS, OK = cabi.TSKV_ERR_INVALID_ARG, cabi.TSKV_ERR_UNSUPPORTED, cabi.TSKV_OK
        inc = lambda cid=1, pt=I64: PushedAggregate(cid, pt, ["increase"])
        gq = lambda cols, **kw: grid_query(truth, columns=cols, group_by_series=True, **kw)
        assert status(gq([inc()] * 8)) == OK
        assert status(gq([inc()] * 9)) == INV
        assert status(gq([inc(5, cabi.TSKV_PT_BOOL)])) == INV
        assert status(gq([inc(0, cabi.TSKV_PT_TIME)])) == INV
        assert status(gq([inc(1, 9)])) == INV
        assert status(gq([PushedAggregate(1, I64, ["count"]), inc(1, F64)])) == INV
        assert status(gq([inc(1, I64), inc(1, U64)])) == INV
        assert status(gq([PushedAggregate(1, I64, ["median"]), inc(1, U64)])) == INV
        many = lambda n: [PushedAggregate(100 + i, I64, ["count"]) for i in range(n)] + [inc()] * 8
        assert status(gq(many(110), pairs=[(1, I64, 2, F64)] * 4)) == OK  # 126 columns
        assert status(gq(many(111), pairs=[(1, I64, 2, F64)] * 4)) == INV
        masked = _RawQuery([inc()], first_bucket_start=0, n_buckets=1, group_by_series=True,
                           patch=lambda c: setattr(c, "agg_mask", cabi.TSKV_AGG_COUNT))
        assert prepare_status(masked) == INV
        # cells that could hold two selected series
        assert status(grid_query(truth, columns=[inc()])) == UNS  # ungrouped over the whole page set
        assert status(grid_query(truth, columns=[inc()], series_ids=np.array([0, 1], dtype=np.uint32))) == UNS
        assert status(grid_query(truth, columns=[inc()], series_ids=np.array([1], dtype=np.uint32))) == OK
        q2 = grid_query(truth, columns=[inc()], series_ids=np.array([0, 1, 2], dtype=np.uint32))
        assert status(q2, group_ids=np.array([0, 1, 0], dtype=np.uint32), n_groups=2) == UNS
        assert status(q2, group_ids=np.array([2, 1, 0], dtype=np.uint32), n_groups=3) == OK
        # sliding windows and labelled buckets
        with pytest.raises(ValueError):
            eng.scan_aggregate(pages, gq([inc()]), slide=W // 5)
        assert prepare_status(gq([inc()]), slide=W // 5) == UNS
        edges = np.array([T0 - 10 * STEP, T0 + 20 * STEP, T0 + 100 * STEP], dtype=np.int64)
        ql = grid_query(truth, columns=[inc()], width=0, group_by_series=True)
        ql.n_buckets = 1
        assert status(ql, edges=edges, labels=np.array([0, 0], dtype=np.uint32)) == UNS
        ql.n_buckets = 2
        assert status(ql, edges=edges) == OK
    finally:
        pages.close()


RANK_INPUTS = [pytest.param(n, "plain", id=str(n)) for n in (1, 3, 4, 8)] + \
    [pytest.param(n, kind, id="%d-%s" % (n, kind)) for kind in ("files", "tombstones", "unselected") for n in (3, 4)]


@pytest.mark.parametrize("n, kind", RANK_INPUTS)
def test_ranks(eng, n, kind):
    """Series shards on n ranks, GROUP BY series: the all-gather merge and the all-reduce partials path sum every rank's
    increases; each cell is one rank's, so the result is the whole scan's. Page sets: plain; merge_arena's chunk files
    (merge groups at the start, middle and end of a series); tombstones of rows and of columns; series the query does
    not select, which the "unselected" layout puts alone on rank 0."""
    kw, scan_kw, unselected = {}, {}, ()
    if kind == "files":
        a, d, truth, files = merge_arena(4)
        kw = scan_kw = {"files": files}
    else:
        a, d, truth = arena(7, n_series=10, n_points=300)
    if kind == "tombstones":
        tombs = cabi.tombstones([(3, 2, T0 + 50 * STEP, T0 + 120 * STEP), (5, 1, T0, T0 + 200 * STEP),
                                 (7, None, T0 + 10 * STEP, T0 + 40 * STEP), (None, None, T0 + 250 * STEP, T0 + 260 * STEP)])
        kw, scan_kw = {"tombstones": tombs}, {"tombstones": tombs}
    every = np.array(sorted(truth), dtype=np.uint32)
    if kind == "unselected":
        unselected = every[[0, 5]]
    ids = np.setdiff1d(every, unselected).astype(np.uint32)
    q = grid_query(truth, group_by_series=True, series_ids=ids)
    outs = layouts(every, n, unselected=unselected)
    assert kind != "unselected" or "unselected" in outs
    for name, (shards, order) in outs.items():
        with RankScans(eng, a, d, q, shards, **scan_kw) as rs:
            rs.run()
            for r, res in enumerate(rs.gather(order)):
                check_increases(res, truth, q, "N=%d %s %s gather rank %d" % (n, kind, name, r), **kw)
            for r, res in enumerate(rs.allreduce(order)):
                check_increases(res, truth, q, "N=%d %s %s all-reduce rank %d" % (n, kind, name, r), **kw)


def time_partitions(seed, n_ranks=4, n_series=8, n_rows=600):
    """Every series one run of n_rows rows STEP apart, cut at 1-3 rows inside buckets of W (never on a bucket edge)
    into 2-4 partitions on distinct ranks, each partition one or two column groups. -> (arena, descs, whole truth,
    per-rank truths, per-rank descriptor masks)."""
    rng = np.random.default_rng(seed)
    b = datagen.ArenaBuilder()
    truth, ranks, cg_rank = {}, [dict() for _ in range(n_ranks)], []
    per_bucket = W // STEP
    for sid in range(n_series):
        ts = T0 + np.arange(n_rows, dtype=np.int64) * STEP
        p = int(rng.integers(2, n_ranks + 1))
        cuts = np.sort(rng.choice([k for k in range(20, n_rows - 20) if k % per_bucket], p - 1, replace=False))
        owners = np.sort(rng.choice(n_ranks, p, replace=False))
        cols = {}
        for cid, pt in FIELDS:
            v = np.cumsum(rng.integers(-2, 6, n_rows)).astype(DT[pt]) if pt != U64 else np.cumsum(rng.integers(0, 6, n_rows)).astype(np.uint64)
            cols[cid] = (v + rng.random(n_rows) if pt == F64 else v, rng.random(n_rows) > 0.1)
        bounds = [0] + list(cuts) + [n_rows]
        for k in range(p):
            lo, hi = int(bounds[k]), int(bounds[k + 1])
            split = [lo, (lo + hi) // 2, hi] if rng.random() < 0.5 else [lo, hi]
            for g0, g1 in zip(split, split[1:]):
                part = {cid: (v[g0:g1], ok[g0:g1]) for cid, (v, ok) in cols.items()}
                b.add_column_group(sid, ts[g0:g1], [(cid, pt, part[cid][0], part[cid][1]) for cid, pt in FIELDS])
                ranks[owners[k]].setdefault(sid, []).append((ts[g0:g1], part))
                cg_rank.append(int(owners[k]))
        truth[sid] = [(ts, cols)]
    a, d = b.finish()
    cg_of_desc = np.cumsum(d["phys_type"] == cabi.TSKV_PT_TIME) - 1
    masks = [np.asarray(cg_rank)[cg_of_desc] == r for r in range(n_ranks)]
    return a, d, truth, ranks, masks


def test_ranks_time_partitions(eng):
    """One series split over ranks by time, as time-partitioned vnodes hold it. The reference's increase merges partial
    states by adding them (IncreaseAccumulator::merge_inner, query_server/query/src/extension/expr/aggregate_function/
    increase.rs:109-114), so the pair across a partition boundary is never counted: the expected cell is the wrapping
    sum over ranks of each rank's exact increase (f64: the sum, within the magnitudes' tolerance), valid where any rank's
    is. The scan's all-gather merge and all-reduce partials path sum the increase sections the same way. GROUP BY
    series, and one selected series ungrouped; at least one cell differs from the whole series' increase."""
    a, d, truth, ranks, masks = time_partitions(11)
    ids = np.array(sorted(truth), dtype=np.uint32)
    for what, q in (("series", grid_query(truth, group_by_series=True, series_ids=ids)),
                    ("one series", grid_query(truth, series_ids=ids[3:4]))):
        n_cells = (len(ids) if q.group_by_series else 1) * q.n_buckets
        with RankScans(eng, a, d, q, masks) as rs:
            rs.run()
            results = [("gather", res) for res in rs.gather()] + [("all-reduce", res) for res in rs.allreduce()]
        for k, c in enumerate(INCS):
            parts = [exact_increase_cells(rt, q, c.column_id, c.phys_type, n_cells) for rt in ranks]
            if c.phys_type == F64:
                v = np.sum([p[0].view(np.float64) for p in parts], axis=0).view(np.uint64)
            else:
                v = np.sum([p[0] for p in parts], axis=0, dtype=np.uint64)
            merged = (v, np.any([p[1] for p in parts], axis=0), np.sum([p[2] for p in parts], axis=0))
            whole = exact_increase_cells(truth, q, c.column_id, c.phys_type, n_cells)
            np.testing.assert_array_equal(whole[1], merged[1])
            if c.phys_type != F64:
                assert (whole[0] != merged[0])[merged[1]].any(), (what, k)
            for path, res in results:
                check_increase(res, len(res.names) - len(INCS) + k, merged, c.phys_type,
                               what="time partitions %s %s increase %d" % (what, path, k))


def test_ranks_ungrouped(eng):
    """An ungrouped multi-rank increase decides from the query alone: without series_ids every rank refuses, also when
    each rank holds one series (the exchange would sum several series' increases into one cell); with one selected
    series every rank accepts, and the merged result is that series' increase."""
    a, d, truth = arena(8, n_series=4, n_points=300)
    ids = np.array(sorted(truth), dtype=np.uint32)
    q = grid_query(truth)
    for name, (shards, _) in list(layouts(ids, 4).items()) + [("one each", ([ids[r:r + 1] for r in range(4)], None))]:
        for r, shard in enumerate(shards):
            pages = eng.upload_pages(a, d[np.isin(d["series_id"], shard)])
            try:
                with pytest.raises(TskvError) as e:
                    eng.prepare(pages, multi_rank(q)).close()
                assert e.value.status == cabi.TSKV_ERR_UNSUPPORTED, (name, r)
            finally:
                pages.close()
    q1 = grid_query(truth, series_ids=ids[2:3])
    for name, (shards, order) in layouts(ids, 4).items():
        with RankScans(eng, a, d, q1, shards) as rs:
            rs.run()
            for r, res in enumerate(rs.gather(order)):
                check_increases(res, truth, q1, "ungrouped one series %s gather rank %d" % (name, r))
            for r, res in enumerate(rs.allreduce(order)):
                check_increases(res, truth, q1, "ungrouped one series %s all-reduce rank %d" % (name, r))


def random_case(rng, truth):
    """A random query over `truth` that keeps one series per cell, with its scan keyword arguments and reference ones."""
    ids = np.array(sorted(truth), dtype=np.uint32)
    cols = [PushedAggregate(c, pt, ["increase"] + (["count"] if rng.random() < 0.3 else [])) for c, pt in FIELDS
            if rng.random() < 0.7] or [INCS[0]]
    kw = {}
    if rng.random() < 0.4:
        kw["predicates"] = [(2, F64, "<", float(rng.integers(0, 60)))]
    if rng.random() < 0.4:
        lo = int(rng.integers(0, 200))
        kw["time_ranges"] = [(T0 + lo * STEP, T0 + (lo + int(rng.integers(20, 200))) * STEP)]
    width = int(rng.choice([0, 5 * STEP, W, 4 * W]))
    grouping = rng.choice(["series", "tags", "one"])
    scan_kw, ref_kw = {}, {}
    if grouping == "one":
        q = grid_query(truth, columns=cols, width=width, series_ids=ids[int(rng.integers(0, len(ids))):][:1], **kw)
    else:
        sel = np.sort(rng.choice(ids, size=int(rng.integers(1, len(ids) + 1)), replace=False)).astype(np.uint32)
        q = grid_query(truth, columns=cols, width=width, series_ids=sel, group_by_series=grouping == "series", **kw)
        if grouping == "tags":
            gids = rng.permutation(len(sel)).astype(np.uint32)
            scan_kw = dict(group_ids=gids, n_groups=len(sel))
            ref_kw = dict(group_ids=gids)
    return q, scan_kw, ref_kw


def test_random_combinations_twice(eng):
    """100 seeded random queries, each scanned twice: the integer outputs are byte-identical and every output meets the
    reference."""
    for arena_seed in range(4):
        a, d, truth = arena(100 + arena_seed, n_series=6, n_points=250, jitter=200 if arena_seed % 2 else 0,
                            raw_frac=0.3 if arena_seed == 3 else 0.0)
        pages = eng.upload_pages(a, d)
        try:
            rng = np.random.default_rng(arena_seed)
            for case in range(25):
                q, scan_kw, ref_kw = random_case(rng, truth)
                what = "arena %d case %d" % (arena_seed, case)
                r1 = eng.scan_aggregate(pages, q, **scan_kw)
                r2 = eng.scan_aggregate(pages, q, **scan_kw)
                for j, (cid, agg) in enumerate(r1.names):
                    if agg == "increase" and r1.phys[cid] != F64:
                        np.testing.assert_array_equal(r1.values[j], r2.values[j], err_msg=what)
                        np.testing.assert_array_equal(r1.validity[j], r2.validity[j], err_msg=what)
                check_increases(r1, truth, q, what, min_valid=0, **ref_kw)
        finally:
            pages.close()


def test_golden_test_increase_grouped(eng):
    """increase.slt's two series through a grouped scan: 7 and 7."""
    g = load_golden()["test_increase"]
    b = datagen.ArenaBuilder()
    for sid, s in enumerate(g["series"]):
        ts = np.array([np.datetime64(r["time"].replace(" ", "T"), "ns").astype(np.int64) for r in s["rows"]], dtype=np.int64)
        b.add_column_group(sid, ts, [(1, I64, np.array([r["f0"] for r in s["rows"]], dtype=np.int64), None)])
    a, d = b.finish()
    pages = eng.upload_pages(a, d)
    try:
        r = eng.scan_aggregate(pages, QueryOption([PushedAggregate(1, I64, ["increase"])], first_bucket_start=0, n_buckets=1),
                               group_ids=np.array([0, 1], dtype=np.uint32), n_groups=2)
    finally:
        pages.close()
    v, ok = r.column(1, "increase")
    assert ok.all() and [int(x) for x in v[:, 0]] == [g["group_by_t0"]["expected"][s["rows"][0]["t0"]] for s in g["series"]]


def test_golden_func_tb2(eng):
    """func_tb2's rows as one series give 3007 / 6008.0 / 80002; as their real series (by tags) an ungrouped scan is
    refused."""
    g = load_golden()
    cols = {"f0": 1, "f1": 2, "f4": 3}
    t = g["tables"]["func_tb2"]
    ts = np.array([int(r[0]) for r in t["rows"]], dtype=np.int64)
    fields = [(cid, golden_tb2(g, name)[2], golden_tb2(g, name)[1], None) for name, cid in cols.items()]
    q = QueryOption([PushedAggregate(cid, pt, ["increase"]) for cid, pt, _, _ in fields], first_bucket_start=0, n_buckets=1)
    b = datagen.ArenaBuilder()
    b.add_column_group(0, ts, fields)
    a, d = b.finish()
    pages = eng.upload_pages(a, d)
    try:
        r = eng.scan_aggregate(pages, q)
    finally:
        pages.close()
    for ans in g["func_tb2"]:
        v, ok = r.column(cols[ans["column"]], "increase")
        assert ok[0, 0] and repr(v[0, 0].item()) == ans["expected"], (ans, v)
    tags = [tuple(row[6:9]) for row in t["rows"]]
    series = {k: i for i, k in enumerate(sorted(set(tags)))}
    b = datagen.ArenaBuilder()
    for key, sid in series.items():
        rows = [i for i, k in enumerate(tags) if k == key]
        b.add_column_group(sid, ts[rows], [(cid, pt, v[rows], None) for cid, pt, v, _ in fields])
    a, d = b.finish()
    pages = eng.upload_pages(a, d)
    try:
        with pytest.raises(TskvError) as e:
            eng.scan_aggregate(pages, q)
        assert e.value.status == cabi.TSKV_ERR_UNSUPPORTED
    finally:
        pages.close()
