"""Column pairs (tskv_query.n_pairs: covar / covar_samp / covar_pop / corr) through the scan, against the exact per-cell
co-moments of tests/covariance_reference.py: every grouping, NULL patterns that differ between x and y, column groups
without y, predicates, tombstones on one operand, time ranges, host-resident pages with CRC on read, overlapping chunk
files, special values, constant columns, C(x, x) against TSKV_AGG_M2, counters, refusals and graph replay (the
multi-rank merge of pairs: tests/test_gpu_multi_rank.py)."""

import ctypes as C

import numpy as np
import pytest

from cnosdb_b200 import cabi, datagen
from cnosdb_b200.engine import Engine, PushedAggregate, QueryOption, TskvError
from tests.covariance_reference import check_pair, exact_pair_cells, load_golden, tb2_column
from tests.exact_arenas import add_column_group, two_file_arena
from tests.helpers import bucket_spec, random_arena

pytestmark = pytest.mark.gpu

I64, U64, F64 = cabi.TSKV_PT_I64, cabi.TSKV_PT_U64, cabi.TSKV_PT_F64
T0, STEP, W = 1_000_000, 1000, 50_000
FIELDS = ((1, I64), (2, F64), (3, U64), (4, F64))
PAIRS = [(1, I64, 2, F64), (2, F64, 3, U64), (3, U64, 1, I64), (2, F64, 2, F64), (4, F64, 1, I64)]


@pytest.fixture(scope="module")
def eng():
    e = Engine(0)
    yield e
    e.close()


def arena(seed, null_frac=0.2, jitter=0, raw_frac=0.0, drop_y=True, n_series=24, n_points=400):
    """random_arena with several column groups per series; with drop_y, every third column group of odd series loses
    column 4 (its pairs have no paired row there)."""
    rng = np.random.default_rng(seed)
    _, _, truth = random_arena(rng, n_series=n_series, n_points=n_points, fields=FIELDS, null_frac=null_frac, t0=T0,
                               step=STEP, jitter=jitter, raw_frac=raw_frac, multi_cg=True)
    b = datagen.ArenaBuilder()
    out = {}
    for sid, cgs in truth.items():
        for k, (ts, cols) in enumerate(cgs):
            if drop_y and sid % 2 and k % 3 == 0:
                cols = {c: v for c, v in cols.items() if c != 4}
            fl = [(c, pt, cols[c][0], None if cols[c][1].all() else cols[c][1]) for c, pt in FIELDS if c in cols]
            b.add_column_group(sid, ts, fl)
            out.setdefault(sid, []).append((ts, cols))
    a, d = b.finish()
    return a, d, out


def grid_query(truth, pairs=PAIRS, columns=(), **kw):
    t_hi = max(int(ts[-1]) for cgs in truth.values() for ts, _ in cgs)
    fbs, nb = bucket_spec(T0 - 10 * STEP, t_hi + STEP, W)
    kw.setdefault("width", W)
    if kw["width"] <= 0:
        fbs, nb = 0, 1
    return QueryOption(list(columns), first_bucket_start=fbs, n_buckets=nb, pairs=pairs, **kw)


def check_all(res, truth, q, what, rtol=1e-9, **kw):
    n_cells = res.n_groups * res.n_buckets
    for k, p in enumerate(q.pairs):
        check_pair(res, k, exact_pair_cells(truth, q, p, n_cells, **kw), rtol=rtol, what="%s pair %d" % (what, k))


@pytest.mark.parametrize("kind", ["rle", "jitter", "raw"])
def test_groupings(eng, kind):
    a, d, truth = arena(1, jitter=300 if kind == "jitter" else 0, raw_frac=0.5 if kind == "raw" else 0.0)
    pages = eng.upload_pages(a, d)
    try:
        sel = np.arange(0, 24, 2, dtype=np.uint32)
        q = grid_query(truth, series_ids=sel)
        check_all(eng.scan_aggregate(pages, q), truth, q, kind + " bucket")
        qs = grid_query(truth, series_ids=sel, group_by_series=True)
        check_all(eng.scan_aggregate(pages, qs), truth, qs, kind + " series")
        qu = grid_query(truth, width=0, time_ranges=[(T0 + 20 * STEP, T0 + 150 * STEP), (T0 + 300 * STEP, T0 + 900 * STEP)])
        check_all(eng.scan_aggregate(pages, qu), truth, qu, kind + " unbucketed, two ranges")
        gids = (sel % 3).astype(np.uint32)
        res = eng.scan_aggregate(pages, q, group_ids=gids, n_groups=3)
        check_all(res, truth, q, kind + " tags", group_ids=gids)
        edges = np.array([T0 - 10 * STEP, T0 + 77 * STEP, T0 + 200 * STEP, T0 + 555 * STEP, T0 + 2000 * STEP], dtype=np.int64)
        qe = grid_query(truth, width=0, series_ids=sel)
        qe.n_buckets = 4
        check_all(eng.scan_aggregate(pages, qe, edges=edges), truth, qe, kind + " edges", edges=edges)
        labels = np.array([1, 0, 1, 0], dtype=np.uint32)
        ql = grid_query(truth, width=0, series_ids=sel)
        ql.n_buckets = 2
        check_all(eng.scan_aggregate(pages, ql, edges=edges, labels=labels), truth, ql, kind + " labels", edges=edges, labels=labels)
    finally:
        pages.close()


def test_filters_tombstones_host_resident(eng):
    a, d, truth = arena(2)
    tombs = cabi.tombstones([(3, 2, T0 + 50 * STEP, T0 + 120 * STEP), (5, 4, T0, T0 + 300 * STEP),
                             (7, None, T0 + 10 * STEP, T0 + 40 * STEP), (None, None, T0 + 600 * STEP, T0 + 610 * STEP)])
    for host in (False, True):
        pages = eng.upload_pages(a, d, host_resident=host, verify_on_read=True)
        try:
            pages.set_tombstones(tombs)
            q = grid_query(truth, predicates=[(1, I64, ">", -40)], time_ranges=[(T0 + 5 * STEP, T0 + 800 * STEP)])
            check_all(eng.scan_aggregate(pages, q), truth, q, "filters host=%s" % host, tombstones=tombs)
        finally:
            pages.close()


def test_outputs_and_counters_unchanged(eng):
    """Other outputs equal the query without pairs; reader counters equal that query with the operands as COUNT columns."""
    a, d, truth = arena(3)
    pages = eng.upload_pages(a, d)
    try:
        cols = [PushedAggregate(1, I64, ["count", "sum", "mean", "min", "max"])]
        q = grid_query(truth, pairs=[(2, F64, 4, F64), (1, I64, 3, U64)], columns=cols, predicates=[(3, U64, ">=", 0)])
        r = eng.scan_aggregate(pages, q)
        c = eng.counters()
        q0 = grid_query(truth, pairs=[], columns=cols, predicates=[(3, U64, ">=", 0)])
        r0 = eng.scan_aggregate(pages, q0)
        for name in q0.output_names():
            v, ok = r.column(*name)
            v0, ok0 = r0.column(*name)
            np.testing.assert_array_equal(ok, ok0)
            np.testing.assert_array_equal(np.where(ok, v, 0).view(np.uint64) if v.dtype != np.float64 else np.where(ok, v, 0),
                                          np.where(ok0, v0, 0).view(np.uint64) if v0.dtype != np.float64 else np.where(ok0, v0, 0))
        qc = grid_query(truth, pairs=[], columns=cols + [PushedAggregate(2, F64, ["count"]), PushedAggregate(4, F64, ["count"]),
                                                         PushedAggregate(3, U64, ["count"])], predicates=[(3, U64, ">=", 0)])
        rc = eng.scan_aggregate(pages, qc)
        cc = eng.counters()
        for k in ("page_read_count", "page_read_bytes", "points_decoded", "rows_in_range", "pruned_page_count"):
            assert c[k] == cc[k], k
        assert c["kernel_launches"] > cc["kernel_launches"]
        # n is at most either operand's COUNT
        n, _ = r.pair(0, "n")
        c2, _ = rc.column(2, "count")
        c4, _ = rc.column(4, "count")
        assert (n <= np.minimum(c2, c4)).all() and (n < np.minimum(c2, c4)).any()
        check_all(r, truth, q, "with columns")
    finally:
        pages.close()


def test_x_with_itself_matches_m2(eng):
    a, d, truth = arena(4)
    pages = eng.upload_pages(a, d)
    try:
        q = grid_query(truth, pairs=[(2, F64, 2, F64), (1, I64, 1, I64)],
                       columns=[PushedAggregate(2, F64, ["m2"]), PushedAggregate(1, I64, ["m2"])])
        r = eng.scan_aggregate(pages, q)
        for k, col in enumerate((2, 1)):
            m2, ok = r.column(col, "m2")
            for name in ("c", "m2x", "m2y"):
                v, vok = r.pair(k, name)
                np.testing.assert_array_equal(vok, ok)
                np.testing.assert_allclose(v[ok], m2[ok], rtol=1e-12, atol=1e-300)
    finally:
        pages.close()


def special_arena():
    """Extremes and special values: u64 near 2^63 against i64 extremes, an ill-conditioned f64 column (1e9 + small),
    a constant column, NaN and inf in series 2 only."""
    b = datagen.ArenaBuilder()
    truth = {}
    rng = np.random.default_rng(7)
    n = 300
    for sid in range(4):
        ts = T0 + np.arange(n, dtype=np.int64) * STEP
        x = (np.uint64(2**63 - 5000) + rng.integers(0, 4000, n).astype(np.uint64))
        y = rng.integers(-2**62, 2**62, n).astype(np.int64)
        y[::37] = np.iinfo(np.int64).min
        y[1::41] = np.iinfo(np.int64).max
        z = 1e9 + rng.random(n) * 1e-3
        k = np.full(n, 42.5)
        if sid == 2:
            z[10] = np.nan
            k[20] = np.inf
        fl = [(1, U64, x, None), (2, I64, y, None), (3, F64, z, None), (4, F64, k, None)]
        b.add_column_group(sid, ts, fl)
        truth[sid] = [(ts, {c: (v, np.ones(n, dtype=bool)) for c, _, v, _ in fl})]
    a, d = b.finish()
    return a, d, truth


def test_extremes_special_values_constant(eng):
    a, d, truth = special_arena()
    pages = eng.upload_pages(a, d)
    try:
        pairs = [(1, U64, 2, I64), (3, F64, 1, U64), (4, F64, 3, F64), (4, F64, 4, F64)]
        q = grid_query(truth, pairs=pairs, group_by_series=True)
        r = eng.scan_aggregate(pages, q)
        check_all(r, truth, q, "extremes", rtol=1e-6)
        corr, ok = r.pair(2, "corr")
        # constant x: M2x is exactly 0 and corr exactly 0.0, except where the column holds inf (series 2: NaN)
        m2x, _ = r.pair(2, "m2x")
        for g in (0, 1, 3):
            assert (m2x[g][ok[g]] == 0.0).all() and (corr[g][ok[g]] == 0.0).all()
        assert np.isnan(m2x[2][ok[2]]).any()
        cc, okc = r.pair(3, "corr")
        assert (cc[[0, 1, 3]][okc[[0, 1, 3]]] == 0.0).all()
    finally:
        pages.close()


def test_overlapping_chunk_files(eng):
    """Two overlapping chunk files per series: the pair passes run over the merged rows."""
    a, d, truth, files, _ = two_file_arena(T0, STEP)
    pages = eng.upload_pages(a, d)
    try:
        pages.set_chunk_files(files)
        q = grid_query(truth, pairs=[(1, I64, 2, F64)], group_by_series=True)
        check_all(eng.scan_aggregate(pages, q), truth, q, "overlap", files=files)
    finally:
        pages.close()


class _MaskedOperand(QueryOption):
    """A query whose first pair operand carries a non-zero agg_mask (engine.QueryOption always writes 0 there)."""

    def to_c(self):
        q = super().to_c()
        q.columns[len(self.columns)].agg_mask = cabi.TSKV_AGG_COUNT
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
        INV, UNS = cabi.TSKV_ERR_INVALID_ARG, cabi.TSKV_ERR_UNSUPPORTED
        assert status(grid_query(truth, pairs=[(1, I64, 2, F64)] * 8)) == cabi.TSKV_OK
        assert status(grid_query(truth, pairs=[(1, I64, 2, F64)] * 9)) == INV
        assert status(grid_query(truth, pairs=[(5, cabi.TSKV_PT_BOOL, 2, F64)])) == INV
        assert status(grid_query(truth, pairs=[(1, I64, 0, cabi.TSKV_PT_TIME)])) == INV
        assert status(grid_query(truth, pairs=[(1, I64, 2, 9)])) == INV
        assert status(grid_query(truth, pairs=[(1, F64, 2, F64)], columns=[PushedAggregate(1, I64, ["count"])])) == INV
        assert status(grid_query(truth, pairs=[(1, I64, 2, F64), (1, U64, 2, F64)])) == INV
        assert status(grid_query(truth, pairs=[(1, I64, 2, F64)] * 8,
                                 columns=[PushedAggregate(100 + i, I64, ["count"]) for i in range(111)])) == INV
        masked = _MaskedOperand([], first_bucket_start=0, n_buckets=1, pairs=[(1, I64, 2, F64)])
        assert status(masked) == INV
        # pages of another type under an operand's id: the work-list walk reports it when the scan runs
        assert status(grid_query(truth, pairs=[(1, F64, 2, F64)])) == INV
        # sliding windows: the engine refuses before the library, and the library refuses on its own
        with pytest.raises(ValueError):
            eng.scan_aggregate(pages, grid_query(truth, pairs=[(1, I64, 2, F64)]), slide=W // 5)
        q = grid_query(truth, pairs=[(1, I64, 2, F64)]).to_c()
        h = C.c_void_p()
        assert eng.lib.tskvgpu_scan_prepare_sliding(eng.ctx, pages.handle, C.byref(q), W // 5, C.byref(h)) == UNS
        assert not h.value
        s = eng.prepare(pages, grid_query(truth, pairs=[(1, I64, 2, F64)]))
        try:
            s.run()
            with pytest.raises(TskvError) as e:
                s.partials()
            assert e.value.status == UNS
        finally:
            s.close()
    finally:
        pages.close()


def test_graph_replay(eng, monkeypatch, capfd):
    """tskvgpu_scan_enqueue captures the pass (both pair passes included) into a CUDA graph on its second call and
    replays it from then on; the replayed results meet the exact reference and the capture did not fall back."""
    monkeypatch.setenv("TSKV_DEBUG_BINS", "1")  # (a failed capture says so on stderr)
    a, d, truth = arena(6)
    q = grid_query(truth, pairs=[(1, I64, 2, F64), (4, F64, 3, U64)], group_by_series=True)
    pages = eng.upload_pages(a, d)
    try:
        s = eng.prepare(pages, q)
        try:
            for _ in range(4):
                s.enqueue()
                s.sync()
            res = s.finalize()
            check_all(res, truth, q, "graph replay")
        finally:
            s.close()
    finally:
        pages.close()
    assert "graph capture failed" not in capfd.readouterr().err


# ---- the reference's goldens through the scan --------------------------------------------------------------------------
TB2_IDS = {"f0": (1, U64), "f1": (2, F64), "f4": (5, I64), "-f1": (6, F64)}
ONE, TWO = (7, I64), (8, I64)


def test_goldens_func_tb2(eng):
    """corr.slt / covar*.slt over func_tb2 stored as an arena: f0 (u64), f1 (f64), f4 (i64), -f1 as a column of its own,
    and the constants 1 and 2 as columns (F(1, 2))."""
    g = load_golden()
    rows = g["tables"]["func_tb2"]["rows"]
    ts = np.array([int(r[0]) for r in rows], dtype=np.int64)
    b = datagen.ArenaBuilder()
    fields = [(cid, pt, tb2_column(g, name), None) for name, (cid, pt) in TB2_IDS.items()]
    fields += [(ONE[0], I64, np.ones(len(rows), dtype=np.int64), None), (TWO[0], I64, np.full(len(rows), 2, dtype=np.int64), None)]
    b.add_column_group(0, ts, sorted(fields, key=lambda f: f[0]))
    a, d = b.finish()
    combos = sorted({(c["x"], c["y"]) for c in g["checks"]})
    pairs = [TB2_IDS[x] + TB2_IDS[y] for x, y in combos] + [ONE + TWO]
    q = QueryOption([], first_bucket_start=0, n_buckets=1, pairs=pairs)
    pages = eng.upload_pages(a, d)
    try:
        r = eng.scan_aggregate(pages, q)
    finally:
        pages.close()
    for c in g["checks"]:
        v, ok = r.pair(combos.index((c["x"], c["y"])), c["func"])
        assert ok[0, 0] and abs(v[0, 0] - c["value"]) < c["tolerance"], (c, v)
    for c in g["constants"]:
        v, ok = r.pair(len(combos), c["func"])
        assert ok[0, 0] and v[0, 0] == float(c["expected"]), (c, v)


def test_goldens_unorder_exact_zero(eng):
    """unorderdata_func.slt: the exact covariance is 0; the scan gives exactly 0.0 for corr / covar / covar_pop /
    covar_samp, within an absolute tolerance of the reference's rounding residues (6.28e-17, 4.93e-17, 4.44e-17)."""
    g = load_golden()["unorder"]
    ts = np.array([np.datetime64(r[0].replace(" ", "T"), "ns").astype(np.int64) for r in g["rows"]], dtype=np.int64)
    x = np.array([float(r[1]) for r in g["rows"]])
    y = np.array([float(r[2]) for r in g["rows"]])
    b = datagen.ArenaBuilder()
    b.add_column_group(0, ts, [(1, F64, x, None), (2, F64, y, None)])
    a, d = b.finish()
    pages = eng.upload_pages(a, d)
    try:
        r = eng.scan_aggregate(pages, QueryOption([], first_bucket_start=0, n_buckets=1, pairs=[(1, F64, 2, F64)]))
    finally:
        pages.close()
    assert r.pair(0, "c")[0][0, 0] == 0.0
    for e in g["expected"]:
        v, ok = r.pair(0, e["func"])
        assert ok[0, 0] and v[0, 0] == 0.0 and abs(v[0, 0] - e["value"]) < 1e-16, (e, v)


# ---- every time kind x x value kind x y value kind ------------------------------------------------------------------------
VALUE_KINDS = [(11, I64, None), (12, U64, None), (13, F64, None), (14, I64, datagen.encode_raw), (15, F64, datagen.encode_raw),
               ]


@pytest.mark.parametrize("time_kind", ["rle", "s8b", "raw"])
def test_every_kind_combination(eng, time_kind):
    """All 25 (x kind, y kind) pairs of simple8b i64 / u64, Gorilla f64 and raw i64 / f64 value pages, wide values
    (u64 near 2^63, i64 extremes) and x / y NULLs that differ, over RLE, simple8b (jittered) and raw time pages."""
    rng = np.random.default_rng(21)
    b = datagen.ArenaBuilder()
    truth = {}
    for sid in range(6):
        n = int(rng.integers(200, 700))
        ts = T0 + np.arange(n, dtype=np.int64) * STEP
        if time_kind == "s8b":
            ts = ts + rng.integers(-300, 301, n)
        fl, cols = [], {}
        for cid, pt, enc in VALUE_KINDS:
            if pt == F64:
                v = np.cumsum(rng.integers(-3, 4, n)).astype(np.float64) + rng.random(n)
            elif pt == U64:
                v = np.uint64(2**63 - 10_000) + rng.integers(0, 20_000, n).astype(np.uint64)
            else:
                v = rng.integers(-2**62, 2**62, n) if sid % 2 else np.cumsum(rng.integers(-50, 51, n)).astype(np.int64)
                v[::53] = np.iinfo(np.int64).min
            valid = rng.random(n) >= 0.15
            fl.append((cid, pt, v, valid, enc))
            cols[cid] = (v, valid)
        add_column_group(b, sid, ts, fl, raw_time=time_kind == "raw")
        truth[sid] = [(ts, cols)]
    a, d = b.finish()
    combos = [(x[0], x[1], y[0], y[1]) for x in VALUE_KINDS for y in VALUE_KINDS]
    pages = eng.upload_pages(a, d)
    try:
        for i in range(0, len(combos), 8):
            q = grid_query(truth, pairs=combos[i:i + 8], group_by_series=True)
            check_all(eng.scan_aggregate(pages, q), truth, q, "%s kinds %d" % (time_kind, i), rtol=1e-6)
    finally:
        pages.close()


def test_work_list_feeds_the_pair_kernels(eng):
    """The pair passes run on the x operand's work-list buckets: read the work list back and check that they hold x's
    pages for the tumbling and the edge scan, so that k_scan_pair<PASS2, false> and <PASS2, true> (both passes run on
    every scan with pairs) had their pages. (k_merge_pairs_rows<false> / <true> run the merged rows of
    test_overlapping_chunk_files.)"""
    a, d, truth = arena(8)
    q = grid_query(truth, pairs=[(4, F64, 1, I64)])
    edges = np.array([T0 - 10 * STEP, T0 + 300 * STEP, T0 + 2000 * STEP], dtype=np.int64)
    qe = grid_query(truth, width=0, pairs=[(4, F64, 1, I64)])
    qe.n_buckets = 2
    pages = eng.upload_pages(a, d)
    try:
        for query, kw in ((q, {}), (qe, {"edges": edges})):
            s = eng.prepare(pages, query, **kw)
            try:
                s.run()
                wl = s.work_list()
                res = s.finalize()
            finally:
                s.close()
            n_cols = wl["fill"].size // (2 * 13)  # N_BINS * WL_SUB buckets per column; x (column 4) is column 0
            x_items = sum(int(wl["fill"][(b * n_cols + 0) * 2 + k]) for b in range(13) for k in range(2))
            assert n_cols == 2 and x_items == int((d["column_id"] == 4).sum())
            items = [i for b in range(13) for k in range(2) for key in [(b * n_cols + 0) * 2 + k]
                     for i in range(int(wl["region_start"][key]), int(wl["region_start"][key] + wl["fill"][key]))]
            assert (wl["work_qcol"][items] & 0x7F == 0).all()
            assert sorted(wl["work_page"][items]) == sorted(np.nonzero(d["column_id"] == 4)[0])
            check_all(res, truth, query, "work list", **kw)
    finally:
        pages.close()
