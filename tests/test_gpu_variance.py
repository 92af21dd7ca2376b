"""TSKV_AGG_M2 (the variance state: sum of squared deviations from the cell mean) through the fused scan's two passes.

1. The reference's statistical_agg rows (tests/golden/stat_agg_slt.json) through the scan: var* / stddev* within the .slt
   thresholds; BOOL columns refused like SUM.
2. Every bin kind (RLE, jittered simple8b and raw / NULL time pages; simple8b, narrow, Gorilla and generic value pages;
   short and long pages) with value NULLs, predicates, tombstones, CRC on read, a host-resident page set and overlapping
   chunk files, against the exact M2 (tests/variance_reference.py) at relative 1e-9.
3. GROUP BY bucket, series, tags, edges, labels and unbucketed.
4. An ill-conditioned arena (1e9 + noise of 1e-3) within 1e-6 relative; NaN / +-inf give NaN; cells of 0 and 1 values.
5. Every other output and the reader counters equal those of the same query without M2.
6. Refusals, a two-shard exchange against the single-rank result, graph replay."""
import copy
import datetime
import math

import numpy as np
import pytest

from cnosdb_b200 import cabi, datagen
from cnosdb_b200.engine import STAT_AGGS, PushedAggregate, QueryOption, TskvError
from tests.edges_reference import exact_aggregate_edges
from tests.group_reference import exact_aggregate_grouped
from tests.helpers import bucket_spec, exact_aggregate, random_arena
from tests.labels_reference import exact_aggregate_labels
from tests.test_gpu_bucket_edges import edge_query, random_edges, span
from tests.test_gpu_bucket_labels import label_query
from tests.test_gpu_parity import random_tombstones
from tests.variance_reference import check_m2, exact_m2, with_m2

pytestmark = pytest.mark.gpu

FIELDS = ((1, cabi.TSKV_PT_I64), (2, cabi.TSKV_PT_F64), (3, cabi.TSKV_PT_U64))
AGGS = ("count", "mean", "m2")
COUNTERS = ("points_decoded", "rows_in_range", "page_read_count", "page_read_bytes", "pruned_page_count")


def m2_query(fields=FIELDS, aggs=AGGS, **kw):
    return QueryOption([PushedAggregate(c, pt, aggs) for c, pt in fields], **kw)


def without_m2(q):
    """The same query with M2 taken out of every column."""
    out = copy.copy(q)
    out.columns = [PushedAggregate(c.column_id, c.phys_type, c.agg_mask & ~cabi.TSKV_AGG_M2) for c in q.columns]
    out._keep = None
    return out


def check_rest_unchanged(engine, pages, q, got, counters, what, **kw):
    """Every output but m2, and the reader counters, equal those of the same query without M2: bit for bit, except f64
    sums and means, which the scan adds with atomics in an order that may differ from run to run (within 1e-12)."""
    base = engine.scan_aggregate(pages, without_m2(q), **kw)
    c = engine.counters()
    phys = {col.column_id: col.phys_type for col in q.columns}
    for j, name in enumerate(base.names):
        k = got.names.index(name)
        assert (got.validity[k] == base.validity[j]).all(), "%s %s validity" % (what, name)
        if name[1] == "mean" or (name[1] == "sum" and phys[name[0]] == cabi.TSKV_PT_F64):
            a, b = got.values[k].view(np.float64), base.values[j].view(np.float64)
            assert np.allclose(a, b, rtol=1e-12, atol=0, equal_nan=True), "%s %s values" % (what, name)
        else:
            assert (got.values[k] == base.values[j]).all(), "%s %s values" % (what, name)
    for k in COUNTERS:
        assert counters[k] == c[k], "%s counter %s: %s with M2, %s without" % (what, k, counters[k], c[k])


def scan_and_check(engine, pages, truth, q, what, run_ref, rest=True, **kw):
    got = engine.scan_aggregate(pages, q, **kw)
    counters = engine.counters()
    exp = run_ref()
    check_m2(got, exp, what)
    if rest:
        check_rest_unchanged(engine, pages, q, got, counters, what, **kw)
    return got


# ---- 1. the reference's rows ---------------------------------------------------------------------------------------
def _golden():
    import json
    import os
    with open(os.path.join(os.path.dirname(__file__), "golden", "stat_agg_slt.json")) as f:
        return json.load(f)


GOLDEN = _golden()
GOLDEN_PT = {"BIGINT": cabi.TSKV_PT_I64, "BIGINT UNSIGNED": cabi.TSKV_PT_U64, "DOUBLE": cabi.TSKV_PT_F64,
             "BOOLEAN": cabi.TSKV_PT_BOOL}


def _time_ns(v):
    if v.lstrip("-").isdigit():
        return int(v)
    d = datetime.datetime.strptime(v, "%Y-%m-%d %H:%M:%S.%f").replace(tzinfo=datetime.timezone.utc)
    return int(round(d.timestamp() * 1000)) * 10**6


def golden_arena(table):
    """The table's rows as pages: one series per tag set, its rows in time order; numeric and boolean fields."""
    t = GOLDEN["tables"][table]
    cols = t["columns"]
    fields = [(i + 1, c, GOLDEN_PT[t["types"][c]]) for i, c in enumerate(cols) if c in t["types"] and t["types"][c] in GOLDEN_PT]
    tags = [j for j, c in enumerate(cols) if c.startswith("t") and c != "time"]
    series = {}
    for r in t["rows"]:
        series.setdefault(tuple(r[j] for j in tags), []).append(r)
    b = datagen.ArenaBuilder()
    for sid, key in enumerate(sorted(series)):
        rows = sorted(series[key], key=lambda r: _time_ns(r[0]))
        ts = np.array([_time_ns(r[0]) for r in rows], dtype=np.int64)
        fl = []
        for col_id, c, pt in fields:
            j = cols.index(c)
            if pt == cabi.TSKV_PT_F64:
                v = np.array([float(r[j]) for r in rows], dtype=np.float64)
            elif pt == cabi.TSKV_PT_BOOL:
                v = np.array([r[j] == "true" for r in rows], dtype=np.uint64)
            elif pt == cabi.TSKV_PT_U64:
                v = np.array([int(r[j]) for r in rows], dtype=np.uint64)
            else:
                v = np.array([int(r[j]) for r in rows], dtype=np.int64)
            fl.append((col_id, pt, v, None, None))
        b.add_column_group(sid, ts, fl)
    arena, descs = b.finish()
    return arena, descs, {c: (col_id, pt) for col_id, c, pt in fields}


@pytest.mark.parametrize("table", ["func_tbl", "func_tb2"])
def test_golden_rows(engine, table):
    arena, descs, fields = golden_arena(table)
    pages = engine.upload_pages(arena, descs)
    checks = [c for c in GOLDEN["checks"] if c["table"] == table]
    cols = sorted({c["column"] for c in checks})
    q = QueryOption([PushedAggregate(fields[c][0], fields[c][1], ["count", "m2"] + list(STAT_AGGS)) for c in cols])
    r = engine.scan_aggregate(pages, q)
    for c in checks:
        v, ok = r.column(fields[c["column"]][0], c["func"])
        assert ok[0, 0] and abs(v[0, 0] - c["value"]) < c["tolerance"], (c["src"], v[0, 0])
    for ref in GOLDEN["refused"]:
        if ref["table"] == table and ref["column"] in fields and fields[ref["column"]][1] == cabi.TSKV_PT_BOOL:
            col_id, pt = fields[ref["column"]]
            with pytest.raises(TskvError) as e:
                engine.scan_aggregate(pages, QueryOption([PushedAggregate(col_id, pt, [ref["func"]])]))
            assert e.value.status == cabi.TSKV_ERR_INVALID_ARG
    pages.close()


# ---- 2. bins and read paths ------------------------------------------------------------------------------------------
def bins_arena(kind, n_points):
    rng = np.random.default_rng({"rle": 1, "jitter": 2, "raw": 3}[kind] * 100 + n_points)
    return random_arena(rng, n_series=70, n_points=n_points, fields=FIELDS, null_frac=0.1,
                        jitter=200 if kind == "jitter" else 0, raw_frac=0.3 if kind == "raw" else 0.05, multi_cg=True)


def grid(truth, width):
    lo, hi = span(truth)
    return bucket_spec(lo - 1, hi + 1, width)


@pytest.mark.parametrize("n_points", [300, 2000])
@pytest.mark.parametrize("kind", ["rle", "jitter", "raw"])
def test_bins(engine, kind, n_points, monkeypatch):
    arena, descs, truth = bins_arena(kind, n_points)
    fbs, nb = grid(truth, 37_000)
    lo, hi = span(truth)
    for parts, smem_kb in (("1", None), ("3", None), ("1", "0")):  # TSKV_SMEM_TABLE_KB=0: the global-memory table
        monkeypatch.setenv("TSKV_PARTS", parts)
        if smem_kb is not None:
            monkeypatch.setenv("TSKV_SMEM_TABLE_KB", smem_kb)
        pages = engine.upload_pages(arena, descs)
        q = m2_query(width=37_000, first_bucket_start=fbs, n_buckets=nb)
        scan_and_check(engine, pages, truth, q, "%s/%d parts %s smem_kb %s" % (kind, n_points, parts, smem_kb),
                       lambda: with_m2(lambda: exact_aggregate(truth, q), q))
        q = m2_query(width=37_000, first_bucket_start=fbs, n_buckets=nb, time_ranges=[(lo + 5_000, hi - 7_000)],
                     predicates=[(1, cabi.TSKV_PT_I64, ">", -40)])
        scan_and_check(engine, pages, truth, q, "%s/%d ranges + predicate" % (kind, n_points),
                       lambda: with_m2(lambda: exact_aggregate(truth, q), q))
        tombs = random_tombstones(np.random.default_rng(5), descs, lo, hi)
        pages.set_tombstones(tombs)
        q = m2_query(width=37_000, first_bucket_start=fbs, n_buckets=nb)
        scan_and_check(engine, pages, truth, q, "%s/%d tombstones" % (kind, n_points),
                       lambda: with_m2(lambda: exact_aggregate(truth, q, tombstones=tombs), q))
        pages.close()


@pytest.mark.parametrize("mode", ["host_resident", "verify_on_read"])
def test_read_paths(engine, mode):
    arena, descs, truth = bins_arena("jitter", 1500)
    fbs, nb = grid(truth, 50_000)
    pages = engine.upload_pages(arena, descs, host_resident=mode == "host_resident", verify_on_read=mode == "verify_on_read")
    q = m2_query(width=50_000, first_bucket_start=fbs, n_buckets=nb, series_ids=np.arange(0, 70, 2, dtype=np.uint32))
    scan_and_check(engine, pages, truth, q, mode, lambda: with_m2(lambda: exact_aggregate(truth, q), q))
    pages.close()


def overlap_arena(seed):
    """Per series two files whose column groups overlap in time on a shared 1000-step grid, 20 % NULLs."""
    rng = np.random.default_rng(seed)
    b = datagen.ArenaBuilder()
    truth, files = {}, []
    for sid in range(30):
        for f in (1, 2):
            start = int(rng.integers(0, 200))
            n = int(rng.integers(50, 300))
            ts = 1_000_000 + (start + np.sort(rng.choice(np.arange(2 * n), n, replace=False))).astype(np.int64) * 1000
            fl, cols = [], {}
            for col, pt in FIELDS:
                valid = rng.random(n) >= 0.2
                if pt == cabi.TSKV_PT_F64:
                    v = np.cumsum(rng.integers(-3, 4, n)).astype(np.float64) + rng.random(n)
                elif pt == cabi.TSKV_PT_U64:
                    v = np.cumsum(rng.integers(0, 5, n)).astype(np.uint64) + np.uint64(2**63 - 100)
                else:
                    v = np.cumsum(rng.integers(-50, 51, n)).astype(np.int64)
                fl.append((col, pt, v, valid, datagen.encode_raw if f == 2 and sid % 3 == 0 else None))
                cols[col] = (v, valid)
            b.add_column_group(sid, ts, fl)
            truth.setdefault(sid, []).append((ts, cols))
            files.append(f)
    arena, descs = b.finish()
    return arena, descs, truth, np.array(files, dtype=np.uint64)


def test_overlapping_chunk_files(engine):
    arena, descs, truth, files = overlap_arena(9)
    pages = engine.upload_pages(arena, descs)
    pages.set_chunk_files(files)
    fbs, nb = grid(truth, 20_000)
    for gbs in (False, True):
        q = m2_query(width=20_000, first_bucket_start=fbs, n_buckets=nb, group_by_series=gbs)
        scan_and_check(engine, pages, truth, q, "overlap gbs=%s" % gbs,
                       lambda: with_m2(lambda: exact_aggregate(truth, q, files=files), q))
    pages.close()


# ---- 3. GROUP BY shapes ----------------------------------------------------------------------------------------------
def test_group_by_shapes(engine):
    arena, descs, truth = bins_arena("rle", 1200)
    pages = engine.upload_pages(arena, descs)
    fbs, nb = grid(truth, 45_000)
    lo, hi = span(truth)
    ids = np.arange(3, 70, dtype=np.uint32)
    q = m2_query(series_ids=ids)
    scan_and_check(engine, pages, truth, q, "unbucketed", lambda: with_m2(lambda: exact_aggregate(truth, q), q))
    q = m2_query(width=45_000, first_bucket_start=fbs, n_buckets=nb, series_ids=ids, group_by_series=True)
    scan_and_check(engine, pages, truth, q, "GROUP BY series", lambda: with_m2(lambda: exact_aggregate(truth, q), q))
    gid = (np.arange(ids.size) * 7) % 5
    q = m2_query(width=45_000, first_bucket_start=fbs, n_buckets=nb, series_ids=ids)
    scan_and_check(engine, pages, truth, q, "GROUP BY tags",
                   lambda: with_m2(lambda: exact_aggregate_grouped(truth, q, gid, 5), q, n_groups=5),
                   group_ids=gid, n_groups=5)
    e = random_edges(np.random.default_rng(3), lo, hi, 40, narrow=True)
    qe, e = edge_query(m2_query(series_ids=ids), e)
    scan_and_check(engine, pages, truth, qe, "edges", lambda: with_m2(lambda: exact_aggregate_edges(truth, qe, e), qe),
                   edges=e)
    lab = np.arange(e.size - 1) % 6
    ql = label_query(m2_query(series_ids=ids), 6)
    scan_and_check(engine, pages, truth, ql, "labels",
                   lambda: with_m2(lambda: exact_aggregate_labels(truth, ql, e, lab), ql), edges=e, labels=lab)
    pages.close()


# ---- 4. numerics ----------------------------------------------------------------------------------------------------
def test_ill_conditioned(engine):
    """Values 1e9 + noise of ~1e-3: sum(x^2) - sum(x)^2 / n in f64 keeps no digit of M2 there."""
    rng = np.random.default_rng(11)
    b = datagen.ArenaBuilder()
    truth = {}
    for sid in range(40):
        n = 1000
        ts = 1_000_000 + np.arange(n, dtype=np.int64) * 1000
        v = 1e9 + rng.normal(0, 1e-3, n)
        b.add_column_group(sid, ts, [(2, cabi.TSKV_PT_F64, v, None, None)])
        truth[sid] = [(ts, {2: (v, np.ones(n, dtype=bool))})]
    arena, descs = b.finish()
    pages = engine.upload_pages(arena, descs)
    fbs, nb = grid(truth, 100_000)
    for gbs in (False, True):
        q = m2_query(((2, cabi.TSKV_PT_F64),), width=100_000, first_bucket_start=fbs, n_buckets=nb, group_by_series=gbs)
        got = engine.scan_aggregate(pages, q)
        exp = with_m2(lambda: exact_aggregate(truth, q), q)
        check_m2(got, exp, "ill-conditioned gbs=%s" % gbs, rtol=1e-6)
        j = got.names.index((2, "m2"))
        ok = exp.validity[j]
        naive = []  # the one-pass formula on the same cells loses it all (what the test guards against)
        for sid in range(2):
            x = truth[sid][0][1][2][0][:100]
            naive.append(abs((np.sum(x * x) - np.sum(x) ** 2 / x.size) - exact_m2(x)) / exact_m2(x))
        assert max(naive) > 1e-2 and ok.any()
    pages.close()


def test_special_values_and_small_cells(engine):
    """NaN / +-inf in a cell give NaN; cells with one value read 0.0; empty cells are NULL; huge integers."""
    b = datagen.ArenaBuilder()
    truth = {}
    ts = 1_000_000 + np.arange(8, dtype=np.int64) * 1000  # buckets of 2 rows at width 2000
    f = [np.array([1.0, math.nan, 2.0, 3.0, math.inf, 1.0, -math.inf, math.inf]),
         np.array([0.5, 0.25, 7.0, 7.0, 1e150, -1e150, 3.0, 4.0])]
    iv = [np.array([-2**63, 2**63 - 1, 5, 5, 1, 2, 3, 4], dtype=np.int64),
          np.array([0, 1, 2, 3, 4, 5, 6, 7], dtype=np.int64)]
    uv = np.array([2**64 - 1, 2**63 + 1, 1, 2**64 - 2, 0, 9, 8, 7], dtype=np.uint64)
    valid_one = np.array([True, False, True, True, True, False, False, False])
    for sid in range(2):
        fl = [(1, cabi.TSKV_PT_I64, iv[sid], valid_one if sid else None, None),
              (2, cabi.TSKV_PT_F64, f[sid], None, None), (3, cabi.TSKV_PT_U64, uv, valid_one, None)]
        b.add_column_group(sid, ts, fl)
        truth[sid] = [(ts, {1: (iv[sid], valid_one if sid else np.ones(8, dtype=bool)), 2: (f[sid], np.ones(8, dtype=bool)),
                            3: (uv, valid_one)})]
    arena, descs = b.finish()
    pages = engine.upload_pages(arena, descs)
    q = m2_query(width=2000, first_bucket_start=1_000_000, n_buckets=5, group_by_series=True)
    got = engine.scan_aggregate(pages, q)
    exp = with_m2(lambda: exact_aggregate(truth, q), q)
    check_m2(got, exp, "special values")
    m2, ok = got.column(2, "m2")
    assert np.isnan(m2[0, 0]) and np.isnan(m2[0, 2]) and np.isnan(m2[0, 3]) and not ok[0, 4]
    m2, ok = got.column(3, "m2")  # one value per cell: 0.0; no value: NULL
    assert ok[0, 0] and m2[0, 0] == 0.0 and ok[0, 1] and ok[0, 2] and not ok[0, 3]
    v, ok = got.column(3, "var_samp")
    assert not ok[0, 0] and ok[0, 1]
    pages.close()


# ---- 6. refusals, exchange, replay -----------------------------------------------------------------------------------
def test_refusals(engine):
    arena, descs, truth = bins_arena("rle", 300)
    pages = engine.upload_pages(arena, descs)
    fbs, nb = grid(truth, 40_000)
    q = m2_query(width=40_000, first_bucket_start=fbs, n_buckets=nb)
    with pytest.raises(ValueError):
        engine.scan_aggregate(pages, q, slide=10_000)
    with pytest.raises(ValueError):
        engine.prepare(pages, q, slide=10_000)
    qc = q.to_c()
    import ctypes as C
    h = C.c_void_p()
    for slide in (10_000, 20_000):  # the C ABI: sliding windows refuse M2 before any launch
        st = engine.lib.tskvgpu_scan_prepare_sliding(engine.ctx, pages.handle, C.byref(qc), slide, C.byref(h))
        assert st == cabi.TSKV_ERR_UNSUPPORTED
    s = engine.prepare(pages, q)
    s.run()
    with pytest.raises(TskvError) as e:
        s.partials()
    assert e.value.status == cabi.TSKV_ERR_UNSUPPORTED
    s.close()
    qb = QueryOption([PushedAggregate(1, cabi.TSKV_PT_BOOL, ["m2"])])
    with pytest.raises(TskvError) as e:
        engine.scan_aggregate(pages, qb)
    assert e.value.status == cabi.TSKV_ERR_INVALID_ARG
    pages.close()


def test_two_shard_exchange(engine):
    import torch
    from cnosdb_b200.parallel import device_tensor
    arena, descs, truth = bins_arena("jitter", 800)
    fbs, nb = grid(truth, 60_000)
    ids = np.arange(70, dtype=np.uint32)
    dev = torch.device("cuda", engine.device)
    for gbs in (False, True):
        q = m2_query(width=60_000, first_bucket_start=fbs, n_buckets=nb, series_ids=ids, group_by_series=gbs, multi_rank=True)
        whole = engine.upload_pages(arena, descs)
        single = engine.scan_aggregate(whole, q)
        whole.close()
        exp = with_m2(lambda: exact_aggregate(truth, q), q)
        scans, regions, keep = [], [], []
        for shard in (ids[ids % 2 == 0], ids[ids % 2 == 1]):
            pages = engine.upload_pages(arena, descs[np.isin(descs["series_id"], shard)])
            s = engine.prepare(pages, q)
            s.run()
            ptr, words = s.exchange_view()
            regions.append(device_tensor(ptr, words, torch.int64, dev).clone())
            scans.append(s)
            keep.append(pages)
        gathered = torch.cat(regions)
        torch.cuda.synchronize()
        for s in scans:
            s.merge_gathered(gathered.data_ptr(), 2)
            got = s.finalize()
            check_m2(got, exp, "2-shard exchange gbs=%s" % gbs)
            j = got.names.index((1, "m2"))
            a, b = got.values[j].view(np.float64), single.values[j].view(np.float64)
            assert np.allclose(a, b, rtol=1e-9, atol=0) and (got.validity[j] == single.validity[j]).all()
            s.close()
        for p in keep:
            p.close()


def test_graph_replay(engine):
    arena, descs, truth = bins_arena("rle", 1000)
    pages = engine.upload_pages(arena, descs)
    fbs, nb = grid(truth, 30_000)
    q = m2_query(width=30_000, first_bucket_start=fbs, n_buckets=nb)
    s = engine.prepare(pages, q)
    s.run()
    once = s.finalize()
    launches = engine.counters()["kernel_launches"]
    check_m2(once, with_m2(lambda: exact_aggregate(truth, q), q), "graph replay once")
    for _ in range(4):  # the second enqueue captures both passes as a CUDA graph, the later ones replay it
        s.enqueue()
        s.sync()
        again = s.finalize()
        assert (again.validity == once.validity).all()
        j = once.names.index((2, "m2"))
        assert np.allclose(again.values[j].view(np.float64), once.values[j].view(np.float64), rtol=1e-12, atol=0)
        for name in ((1, "m2"), (3, "m2"), (1, "count"), (2, "count")):
            k = once.names.index(name)
            assert np.allclose(again.values[k].view(np.float64 if name[1] == "m2" else np.uint64).astype(np.float64),
                               once.values[k].view(np.float64 if name[1] == "m2" else np.uint64).astype(np.float64), rtol=1e-12)
    base = engine.prepare(pages, without_m2(q))
    base.run()
    assert launches > engine.counters()["kernel_launches"]  # pass 2 launches kernels of its own
    base.close()
    s.close()
    pages.close()
