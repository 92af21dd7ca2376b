"""Medians (TSKV_QUERY_N_MEDIANS) through the scan, bit for bit against tests/median_reference.py: every grouping over
RLE, jittered and raw time pages with NULLs, predicates, tombstones on the operand, host-resident pages with CRC on read,
overlapping chunk files, keys whose middle ranks part at every digit level, a query that mixes projected aggregates, M2,
a pair and two medians on one column, the counters, every refusal, graph replay and the reference's approx_median.slt
table."""
import ctypes as C

import numpy as np
import pytest

from cnosdb_b200 import cabi, datagen
from cnosdb_b200.engine import Engine, PushedAggregate, QueryOption, TskvError
from tests.exact_arenas import two_file_arena
from tests.helpers import bucket_spec, random_arena
from tests.median_reference import check_median, exact_median_cells
from tests.test_median_reference import golden_column, load_golden

pytestmark = pytest.mark.gpu

I64, U64, F64 = cabi.TSKV_PT_I64, cabi.TSKV_PT_U64, cabi.TSKV_PT_F64
T0, STEP, W = 1_000_000, 1000, 50_000
FIELDS = ((1, I64), (2, F64), (3, U64))
MEDIANS = [PushedAggregate(c, pt, ["median"]) for c, pt in FIELDS]


@pytest.fixture(scope="module")
def eng():
    e = Engine(0)
    yield e
    e.close()


def arena(seed, null_frac=0.2, jitter=0, raw_frac=0.0, n_series=24, n_points=400):
    rng = np.random.default_rng(seed)
    return random_arena(rng, n_series=n_series, n_points=n_points, fields=FIELDS, null_frac=null_frac, t0=T0, step=STEP,
                        jitter=jitter, raw_frac=raw_frac, multi_cg=True)


def grid_query(truth, columns=MEDIANS, **kw):
    t_hi = max(int(ts[-1]) for cgs in truth.values() for ts, _ in cgs)
    fbs, nb = bucket_spec(T0 - 10 * STEP, t_hi + STEP, W)
    kw.setdefault("width", W)
    if kw["width"] <= 0:
        fbs, nb = 0, 1
    return QueryOption(list(columns), first_bucket_start=fbs, n_buckets=nb, **kw)


def check_medians(res, truth, q, what, **kw):
    n_cells = res.n_groups * res.n_buckets
    meds = [c for c in q.columns if c.median]
    assert meds
    for k, c in enumerate(meds):
        exact = exact_median_cells(truth, q, c.column_id, c.phys_type, n_cells, **kw)
        j = len(res.names) - len(meds) + k  # (the median outputs come last, in column order)
        check_median(res, j, exact, what="%s median %d" % (what, k))
        assert exact[1].sum() > 0, what


@pytest.mark.parametrize("kind", ["rle", "jitter", "raw"])
def test_groupings(eng, kind):
    a, d, truth = arena(1, jitter=300 if kind == "jitter" else 0, raw_frac=0.5 if kind == "raw" else 0.0)
    pages = eng.upload_pages(a, d)
    try:
        sel = np.arange(0, 24, 2, dtype=np.uint32)
        q = grid_query(truth, series_ids=sel)
        check_medians(eng.scan_aggregate(pages, q), truth, q, kind + " bucket")
        qs = grid_query(truth, series_ids=sel, group_by_series=True)
        check_medians(eng.scan_aggregate(pages, qs), truth, qs, kind + " series")
        qu = grid_query(truth, width=0, time_ranges=[(T0 + 20 * STEP, T0 + 150 * STEP), (T0 + 300 * STEP, T0 + 900 * STEP)])
        check_medians(eng.scan_aggregate(pages, qu), truth, qu, kind + " unbucketed, two ranges")
        gids = (sel % 3).astype(np.uint32)
        check_medians(eng.scan_aggregate(pages, q, group_ids=gids, n_groups=3), truth, q, kind + " tags", group_ids=gids)
        edges = np.array([T0 - 10 * STEP, T0 + 77 * STEP, T0 + 200 * STEP, T0 + 555 * STEP, T0 + 2000 * STEP], dtype=np.int64)
        qe = grid_query(truth, width=0, series_ids=sel)
        qe.n_buckets = 4
        check_medians(eng.scan_aggregate(pages, qe, edges=edges), truth, qe, kind + " edges", edges=edges)
        labels = np.array([1, 0, 1, 0], dtype=np.uint32)
        ql = grid_query(truth, width=0, series_ids=sel)
        ql.n_buckets = 2
        check_medians(eng.scan_aggregate(pages, ql, edges=edges, labels=labels), truth, ql, kind + " labels", edges=edges,
                      labels=labels)
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
            check_medians(eng.scan_aggregate(pages, q), truth, q, "filters host=%s" % host, tombstones=tombs)
        finally:
            pages.close()


def test_overlapping_chunk_files(eng):
    """Two overlapping chunk files per series: the selection passes run over the merged rows too."""
    a, d, truth, files, _ = two_file_arena(T0, STEP)
    pages = eng.upload_pages(a, d)
    try:
        pages.set_chunk_files(files)
        for gbs in (True, False):
            q = grid_query(truth, columns=MEDIANS[:2], group_by_series=gbs)
            check_medians(eng.scan_aggregate(pages, q), truth, q, "overlap gbs=%s" % gbs, files=files)
    finally:
        pages.close()


def from_ukey(u, pt):
    """The value of type pt whose unsigned order key is u (okey_inv)."""
    k = u ^ (1 << 63)  # the signed key's bit pattern
    if pt == U64:
        return np.uint64(u)
    if pt == I64:
        return np.uint64(k).view(np.int64)
    return np.uint64(k ^ (0x7FFFFFFFFFFFFFFF if k >> 63 else 0)).view(np.float64)


def digit_arena():
    """One series per (type, level L, parity), one bucket: the two middle keys part first at digit L (0: the top 8 bits of
    the unsigned order key), under a common prefix of L digits; the smallest and the largest key of every series are 0
    and 2^64 - 1 (i64 MIN / MAX, f64 -NaN / +NaN), so the extremes share no bit and every case runs 1 + L histogram
    passes, all 8 for L = 7 (keys that differ only in the last digit). Odd cases hold one key more above."""
    b = datagen.ArenaBuilder()
    truth = {}
    rng = np.random.default_rng(5)
    sid = 0
    for cid, pt in FIELDS:
        for L in range(8):
            sh = 8 * (7 - L)
            base = 0xA5A5A5A5A5A5A5A5 & ~((1 << (sh + 8)) - 1) & 0xFFFFFFFFFFFFFFFF
            lo, hi = base | (0x12 << sh) | ((1 << sh) - 1), base | (0x13 << sh)
            keys = [lo - 3 * k for k in range(5)] + [hi + 3 * k for k in range(5)] + [0, (1 << 64) - 1]
            for odd in (False, True):
                ks = keys + ([hi + 100] if odd else [])
                n = len(ks)
                ts = T0 + np.arange(n, dtype=np.int64) * STEP
                v = np.array([from_ukey(k, pt) for k in ks])[rng.permutation(n)]
                v = v.astype({I64: np.int64, U64: np.uint64, F64: np.float64}[pt])
                b.add_column_group(sid, ts, [(cid, pt, v, None)])
                truth[sid] = [(ts, {cid: (v, np.ones(n, dtype=bool))})]
                sid += 1
    a, d = b.finish()
    return a, d, truth


def test_every_digit_level(eng):
    a, d, truth = digit_arena()
    pages = eng.upload_pages(a, d)
    try:
        q = grid_query(truth, columns=[PushedAggregate(1, I64, ["median"]), PushedAggregate(2, F64, ["median"]),
                                       PushedAggregate(3, U64, ["median"])], group_by_series=True)
        res = eng.scan_aggregate(pages, q)
        check_medians(res, truth, q, "digit levels")
        assert eng.counters()["kernel_launches"] >= 17  # prep + 8 x (selection pass, step)
        # every case holds values, and the cells of the series the engine did not ask about are NULL
        for cid, pt in FIELDS:
            v, ok = res.column(cid, "median")
            assert ok.sum() == 16
    finally:
        pages.close()


def test_special_values(eng):
    """NaN of both signs, +-inf, -0.0 / +0.0, i64 / u64 extremes, one value, all values equal."""
    b = datagen.ArenaBuilder()
    truth = {}
    cases = {
        0: (F64, [1.0, np.nan]), 1: (F64, [-np.inf, np.inf]), 2: (F64, [-0.0, 0.0]), 3: (F64, [0.0, -0.0, -0.0]),
        4: (F64, [float(np.uint64(0xFFF8000000000001).view(np.float64)), 1.0, 2.0, np.nan]), 5: (F64, [1e308, 1e308]),
        6: (F64, [2.5]), 7: (F64, [3.25] * 6), 8: (I64, [-3, 0]), 9: (I64, [2**63 - 1] * 2), 10: (I64, [-2**63, 2**63 - 1]),
        11: (I64, [-7] * 5), 12: (U64, [2**64 - 1, 3]), 13: (U64, [2**63, 0, 2**63 + 2, 1]), 14: (F64, [-np.inf, 5.0, np.inf]),
    }
    for sid, (pt, vals) in cases.items():
        cid = {I64: 1, F64: 2, U64: 3}[pt]
        n = len(vals)
        ts = T0 + np.arange(n, dtype=np.int64) * STEP
        v = np.array(vals, dtype={I64: np.int64, U64: np.uint64, F64: np.float64}[pt])
        b.add_column_group(sid, ts, [(cid, pt, v, None)])
        truth[sid] = [(ts, {cid: (v, np.ones(n, dtype=bool))})]
    a, d = b.finish()
    pages = eng.upload_pages(a, d)
    try:
        q = grid_query(truth, group_by_series=True)
        res = eng.scan_aggregate(pages, q)
        check_medians(res, truth, q, "special values")
        v, ok = res.column(1, "median")
        assert (v[8][ok[8]] == -1).all() and (v[9][ok[9]] == -1).all()
        f, _ = res.column(2, "median")
        assert np.isnan(f[0]).any() and np.isnan(f[1]).any() and np.isinf(f[5]).any()
    finally:
        pages.close()


def test_mixed_query_outputs_and_counters(eng):
    """Projected aggregates, M2, a pair and two medians on one column, plus a median of an unprojected column: the other
    outputs equal those of the query without medians; the reader counters equal those of that query with the unprojected
    operand added as a COUNT column."""
    a, d, truth = arena(3)
    pages = eng.upload_pages(a, d)
    try:
        base = [PushedAggregate(1, I64, ["count", "sum", "mean", "min", "max"]), PushedAggregate(2, F64, ["count", "stddev"])]
        with_med = [PushedAggregate(1, I64, ["count", "sum", "mean", "min", "max", "median"]),
                    PushedAggregate(2, F64, ["count", "stddev", "median"]), PushedAggregate(2, F64, ["median"]),
                    PushedAggregate(3, U64, ["median"])]
        kw = dict(pairs=[(1, I64, 2, F64)], predicates=[(3, U64, ">=", 0)], group_by_series=True)
        q = grid_query(truth, columns=with_med, **kw)
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
            if name[1] in ("m2", "c", "m2x", "m2y") or (name[1] in ("sum", "mean") and r.phys.get(name[0]) == F64):
                x, y = x.view(np.float64), y.view(np.float64)  # (f64 sums are added in atomic order)
                np.testing.assert_allclose(x, y, rtol=1e-12, atol=1e-300, err_msg=str(name))
            else:
                np.testing.assert_array_equal(x, y, err_msg=str(name))
        assert len(r.names) == len(names0) + 4 and r.names[-4:] == [(1, "median"), (2, "median"), (2, "median"), (3, "median")]
        np.testing.assert_array_equal(r.values[-3], r.values[-2])
        n_cells = r.n_groups * r.n_buckets
        for j, (cid, pt) in zip((-4, -3, -1), ((1, I64), (2, F64), (3, U64))):
            v_e, ok_e = exact_median_cells(truth, q, cid, pt, n_cells)
            np.testing.assert_array_equal(r.validity[j], ok_e)
            np.testing.assert_array_equal(r.values[j][ok_e], v_e[ok_e], err_msg="median %d" % cid)
        qc = grid_query(truth, columns=base + [PushedAggregate(3, U64, ["count"])], **kw)
        eng.scan_aggregate(pages, qc)
        cc = eng.counters()
        for k in ("page_read_count", "page_read_bytes", "points_decoded", "rows_in_range", "pruned_page_count"):
            assert c[k] == cc[k], k
        assert c["kernel_launches"] >= cc["kernel_launches"] + 17
    finally:
        pages.close()


class _RawQuery(QueryOption):
    """A query whose median operand (the last column entry) is rewritten by `patch` (engine.QueryOption writes agg_mask 0)."""

    def __init__(self, *a, patch=None, flags=0, **kw):
        super().__init__(*a, **kw)
        self.patch, self.flags = patch, flags

    def to_c(self):
        q = super().to_c()
        n = len(self.projected()) + 2 * len(self.pairs) + cabi.query_n_medians(q.reserved) - 1
        if self.patch:
            self.patch(q.columns[n])
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
        med = lambda cid=1, pt=I64: PushedAggregate(cid, pt, ["median"])
        assert status(grid_query(truth, columns=[med()] * 8)) == cabi.TSKV_OK
        assert status(grid_query(truth, columns=[med()] * 9)) == INV
        assert status(grid_query(truth, columns=[med(5, cabi.TSKV_PT_BOOL)])) == INV
        assert status(grid_query(truth, columns=[med(0, cabi.TSKV_PT_TIME)])) == INV
        assert status(grid_query(truth, columns=[med(1, 9)])) == INV
        assert status(grid_query(truth, columns=[PushedAggregate(1, I64, ["count"]), med(1, F64)])) == INV
        assert status(grid_query(truth, columns=[med(1, I64), med(1, U64)])) == INV
        assert status(grid_query(truth, columns=[med(2, F64)], pairs=[(2, I64, 1, I64)])) == INV
        many = lambda n: [PushedAggregate(100 + i, I64, ["count"]) for i in range(n)] + [med()] * 8
        assert status(grid_query(truth, columns=many(110), pairs=[(1, I64, 2, F64)] * 4)) == cabi.TSKV_OK  # 126 columns
        assert status(grid_query(truth, columns=many(111), pairs=[(1, I64, 2, F64)] * 4)) == INV
        masked = _RawQuery([med()], first_bucket_start=0, n_buckets=1, patch=lambda c: setattr(c, "agg_mask", cabi.TSKV_AGG_COUNT))
        assert prepare_status(masked) == INV
        # pages of another type under an operand's id: the work-list walk reports it when the scan runs
        assert status(grid_query(truth, columns=[med(1, F64)])) == INV
        # sliding windows and multi-rank scans: the engine refuses before the library, and the library on its own
        with pytest.raises(ValueError):
            eng.scan_aggregate(pages, grid_query(truth, columns=[med()]), slide=W // 5)
        assert prepare_status(grid_query(truth, columns=[med()]), slide=W // 5) == UNS
        with pytest.raises(ValueError):
            eng.scan_aggregate(pages, grid_query(truth, columns=[med()], multi_rank=True, series_ids=np.arange(4, dtype=np.uint32)))
        mr = _RawQuery([med()], first_bucket_start=0, n_buckets=1, flags=cabi.TSKV_QUERY_MULTI_RANK)
        assert prepare_status(mr) == UNS
        # the cell cap: n_medians x n_cells <= 2^22, here through GROUP BY tags over a small arena
        cap = cabi.TSKV_MAX_MEDIAN_CELLS
        gids = np.arange(4, dtype=np.uint32)
        assert status(QueryOption([med()], n_buckets=1), group_ids=gids, n_groups=cap) == cabi.TSKV_OK
        assert status(QueryOption([med()] * 2, n_buckets=1), group_ids=gids, n_groups=cap // 2 + 1) == UNS
        assert status(QueryOption([med()], n_buckets=1), group_ids=gids, n_groups=cap + 1) == UNS
        # the exchange calls
        s = eng.prepare(pages, grid_query(truth, columns=[med()]))
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


def test_graph_replay(eng, monkeypatch, capfd):
    """The second enqueue captures the pass with its selection passes into a CUDA graph and later ones replay it: every
    replay meets the reference (the histograms are left cleared) and the capture did not fall back."""
    monkeypatch.setenv("TSKV_DEBUG_BINS", "1")  # (a failed capture says so on stderr)
    a, d, truth = arena(6)
    q = grid_query(truth, group_by_series=True)
    pages = eng.upload_pages(a, d)
    try:
        s = eng.prepare(pages, q)
        try:
            for _ in range(4):
                s.enqueue()
                s.sync()
                check_medians(s.finalize(), truth, q, "graph replay")
        finally:
            s.close()
    finally:
        pages.close()
    assert "graph capture failed" not in capfd.readouterr().err


def test_golden_approx_median_table(eng):
    """approx_median.slt's test_approx_median_tbl stored as an arena: median(d_val) = 1.17, median(val) = 4,
    median(u_val) = 2."""
    g = load_golden()
    t = g["table"]
    ts = np.array([np.datetime64(r[0].replace(" ", "T"), "ns").astype(np.int64) for r in t["rows"]], dtype=np.int64)
    ids = {"val": 1, "d_val": 2, "u_val": 3}
    fl = []
    for name, cid in ids.items():
        pt, v, ok = golden_column(g, name)
        fl.append((cid, pt, v, None if ok.all() else ok))
    b = datagen.ArenaBuilder()
    b.add_column_group(0, ts, fl)
    a, d = b.finish()
    pages = eng.upload_pages(a, d)
    try:
        r = eng.scan_aggregate(pages, QueryOption([PushedAggregate(ids[n], golden_column(g, n)[0], ["median"]) for n in ids],
                                                  first_bucket_start=0, n_buckets=1))
    finally:
        pages.close()
    for c in g["checks"]:
        v, ok = r.column(ids[c["column"]], "median")
        assert ok[0, 0] and repr(v[0, 0].item()) == c["expected"], (c, v)
