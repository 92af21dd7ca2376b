"""Sliding windows on the GPU (tskvgpu_scan_prepare_sliding / tskvgpu_scan_aggregate_sliding): panes one slide wide from
the fused kernels, folded into windows by k_window_combine. Checked against the row-expansion reference
(tests/sliding_reference.py), the reference's time_window.slt outputs, the tumbling scan (slide == window), and the
oracle's tumbling panes folded on the host where the reference cannot model the page set (tombstones, overlapping chunks)."""
import numpy as np
import pytest

from cnosdb_b200 import cabi, datagen
from cnosdb_b200.engine import TskvError, sliding_window_grid
from oracle import pyoracle as orc
from tests.helpers import (ALL_AGGS, ALL_NULL_SERIES, GEOM_AGGS, GEOM_FIELDS, GEOM_SERIES, GEOMETRY_CASES, ReferenceError,
                           _okey, _okey_inv, assert_matches_exact, bucket_spec, geometry_arena, geometry_ranges, make_query,
                           random_arena)
from tests.sliding_reference import expand_aggregate, n_windows_per_row, sliding_fit_grid, sliding_status
from tests.test_gpu_overlap_merge import overlapping_arena
from tests.test_gpu_parity import random_tombstones
from tests.test_sliding_reference import slt_cases, slt_queries

pytestmark = pytest.mark.gpu

ENVS = [("0", "1"), ("0", "3"), ("1", "1"), ("1", "3")]  # (TSKV_COOP, TSKV_PARTS)
FIELDS = ((1, cabi.TSKV_PT_I64), (2, cabi.TSKV_PT_F64), (3, cabi.TSKV_PT_U64))
AGGS = ("count", "sum", "min", "max", "mean")


def _scan(engine, pages, q, slide):
    try:
        return engine.scan_aggregate(pages, q, slide=slide), None
    except TskvError as e:
        return None, e.status


def _identical(a, b, what):
    assert a.names == b.names
    assert (a.validity == b.validity).all() and (a.values == b.values).all(), what


def _ints_equal(a, b, what, rtol=1e-12):
    """COUNT / integer SUM / MIN / MAX (and integer MEAN) bit for bit; f64 SUM / MEAN within rtol (summation order)."""
    assert a.names == b.names
    for j, (col, agg) in enumerate(a.names):
        assert (a.validity[j] == b.validity[j]).all(), "%s: %s %s validity" % (what, col, agg)
        if a.phys[col] == cabi.TSKV_PT_F64 and agg in ("sum", "mean"):
            x, y = a.values[j].view(np.float64), b.values[j].view(np.float64)
            assert np.allclose(x, y, rtol=rtol, atol=0), "%s: %s %s" % (what, col, agg)
        else:
            assert (a.values[j] == b.values[j]).all(), "%s: %s %s" % (what, col, agg)


def test_slide_equal_to_the_window_is_the_tumbling_scan(engine):
    rng = np.random.default_rng(5)
    arena, descs, _ = random_arena(rng, n_series=60, n_points=500, fields=FIELDS, null_frac=0.1, jitter=300, multi_cg=True)
    pages = engine.upload_pages(arena, descs)
    w = 17_000
    fbs, nb = bucket_spec(1_000_000 - 500, 1_000_000 + 1_100_000, w, origin=3)
    for gbs in (False, True):
        q = make_query(FIELDS, ALL_AGGS, width=w, origin=3, first_bucket_start=fbs, n_buckets=nb, group_by_series=gbs)
        _identical(engine.scan_aggregate(pages, q, slide=w), engine.scan_aggregate(pages, q), "slide == width gbs=%s" % gbs)
    pages.close()


@pytest.mark.parametrize("case", slt_cases(), ids=lambda c: c["name"])
def test_slt_goldens(engine, case):
    b = datagen.ArenaBuilder()
    by_series = {}
    for (t, f0, f1), sid in zip(case["rows"], case["series"]):
        by_series.setdefault(sid, []).append((t, f0, f1))
    for sid, rows in sorted(by_series.items()):
        b.add_column_group(sid, np.array([r[0] for r in rows], dtype=np.int64),
                           [(1, cabi.TSKV_PT_I64, np.array([r[1] for r in rows], dtype=np.int64), None),
                            (2, cabi.TSKV_PT_F64, np.array([r[2] for r in rows], dtype=np.float64), None)])
    arena, descs = b.finish()
    pages = engine.upload_pages(arena, descs)
    for q, expect in slt_queries(case):
        got = engine.scan_aggregate(pages, q, slide=case["slide"])
        count, s0, s1 = got.column(1, "count")[0][0], got.column(1, "sum")[0][0], got.column(2, "sum")[0][0]
        for j in range(q.n_buckets):
            rows = expect.get(j, [])
            assert count[j] == len(rows), j
            if rows:
                assert s0[j] == sum(case["rows"][r][1] for r in rows) and s1[j] == sum(case["rows"][r][2] for r in rows), j
    pages.close()


def _slides(w):
    return sorted({s for s in (w // 2, w // 3, (2 * w) // 3 + 1) if 1 <= s < w})


@pytest.mark.parametrize("case", GEOMETRY_CASES, ids=[c[0] for c in GEOMETRY_CASES])
def test_sliding_geometry(engine, case, monkeypatch):
    """The bucket-geometry sweep with windows of the case's width and several slides: COUNT / SUM / MIN / MAX / integer
    MEAN bit-exact against row expansion, f64 within its bound, every refusal and every grid one window short."""
    name, step, w, origin, t0, n, kinds = case
    arena, descs, truth = geometry_arena(len(name), t0, step, n)
    pages = engine.upload_pages(arena, descs)
    few = np.array([0, 1, 40, 41, ALL_NULL_SERIES, 80, 81], dtype=np.uint32)
    for slide in _slides(w):
        for kind in kinds[:2]:
            ranges = geometry_ranges(kind, t0, step, n, w, origin)
            grid = sliding_fit_grid(truth, w, slide, origin, ranges)
            if grid is None:
                continue
            fbs, nb = grid
            g = dict(width=w, origin=origin, first_bucket_start=fbs, n_buckets=nb, time_ranges=ranges)
            queries = [("bucket", make_query(GEOM_FIELDS, GEOM_AGGS, **g)),
                       ("by_series", make_query(GEOM_FIELDS, GEOM_AGGS, group_by_series=True,
                                                series_ids=few if nb * GEOM_SERIES > 300_000 else None, **g)),
                       ("predicate", make_query(GEOM_FIELDS, GEOM_AGGS, predicates=[(1, cabi.TSKV_PT_I64, ">=", 0)], **g))]
            if kind == "none" and nb - 1 >= n_windows_per_row(w, slide):  # one window short at either end
                for f in (fbs + slide, fbs):
                    queries.append(("short@%d" % f, make_query(GEOM_FIELDS, GEOM_AGGS, width=w, origin=origin,
                                                               first_bucket_start=f, n_buckets=nb - 1)))
            for qname, q in queries:
                what = "%s slide=%d %s %s" % (name, slide, kind, qname)
                refusal = sliding_status(truth, q, slide)
                if refusal is not None:
                    assert _scan(engine, pages, q, slide)[1] == refusal, what
                    continue
                try:
                    exp, err = expand_aggregate(truth, q, slide), None
                except ReferenceError as e:
                    exp, err = None, e.status
                if qname.startswith("short"):
                    assert err == cabi.TSKV_ERR_BUCKET_RANGE, what
                for coop, parts in ENVS:
                    monkeypatch.setenv("TSKV_COOP", coop)
                    monkeypatch.setenv("TSKV_PARTS", parts)
                    wh = "%s coop=%s parts=%s" % (what, coop, parts)
                    got, st = _scan(engine, pages, q, slide)
                    assert st == err, "%s: status %s, expected %s" % (wh, st, err)
                    if err is None:
                        assert_matches_exact(got, exp, what=wh)
    pages.close()


def test_refusals(engine):
    rng = np.random.default_rng(8)
    arena, descs, truth = random_arena(rng, n_series=8, n_points=200, fields=FIELDS, t0=-100_000, step=1000)
    pages = engine.upload_pages(arena, descs)
    fbs, nb = sliding_fit_grid(truth, 10_000, 2_000, 0, [])
    base = dict(width=10_000, origin=0, first_bucket_start=fbs, n_buckets=nb)
    cases = [
        (make_query(FIELDS, AGGS, **base), 0, cabi.TSKV_ERR_INVALID_ARG),
        (make_query(FIELDS, AGGS, **base), -2_000, cabi.TSKV_ERR_INVALID_ARG),
        (make_query(FIELDS, AGGS, **dict(base, width=0, n_buckets=1)), 2_000, cabi.TSKV_ERR_INVALID_ARG),
        (make_query(FIELDS, ("count", "first"), **base), 2_000, cabi.TSKV_ERR_UNSUPPORTED),
        (make_query(FIELDS, ("last",), **base), 2_000, cabi.TSKV_ERR_UNSUPPORTED),
        (make_query(FIELDS, AGGS, **base), 10_001, cabi.TSKV_ERR_UNSUPPORTED),
        (make_query(FIELDS, AGGS, **dict(base, width=2**61)), 2**58, cabi.TSKV_ERR_UNSUPPORTED),
        (make_query(FIELDS, AGGS, **base), 99, cabi.TSKV_ERR_INVALID_ARG),                  # k = 102
        (make_query(FIELDS, AGGS, **dict(base, n_buckets=4)), 2_000, cabi.TSKV_ERR_INVALID_ARG),  # n_buckets < k = 5
        (make_query(FIELDS, AGGS, **dict(base, width=2**61 - 1, n_buckets=8)), 2**60 + 1, cabi.TSKV_ERR_INVALID_ARG),  # > 2^63
        (make_query(FIELDS, AGGS, **base), 3_000, cabi.TSKV_ERR_UNSUPPORTED),  # 10000 % 3000 != 0, rows with t < 0
    ]
    for q, slide, status in cases:
        assert sliding_status(truth, q, slide) == status
        assert _scan(engine, pages, q, slide)[1] == status, (slide, status)
        with pytest.raises(TskvError) as e:
            engine.prepare(pages, q, slide=slide)
        assert e.value.status == status
    # the truncating-% rows are not selected: accepted, and equal to row expansion
    q = make_query(FIELDS, AGGS, **dict(base, time_ranges=[(0, 10**9)]))
    assert sliding_status(truth, q, 3_000) is None
    assert_matches_exact(engine.scan_aggregate(pages, q, slide=3_000), expand_aggregate(truth, q, 3_000))
    pages.close()


def fold_panes(panes, k, n_windows):
    """COUNT / SUM / MIN / MAX / f64 MEAN of the windows from a tumbling result over their panes (window j: panes
    j - k + 1 .. j): {(column, agg): (values [groups, windows], validity)}; integer MEAN is left out."""
    out = {}
    n_panes = n_windows - k + 1
    span = [(max(0, j - k + 1), min(j, n_panes - 1) + 1) for j in range(n_windows)]
    for col, agg in panes.names:
        pt = panes.phys[col]
        v, ok = panes.column(col, agg)
        cnt = panes.column(col, "count")[0].astype(np.uint64)
        wc = np.stack([cnt[:, a:b].sum(axis=1) for a, b in span], axis=1)
        have = wc > 0
        if agg == "count":
            out[(col, agg)] = (wc, np.ones_like(have))
        elif agg == "sum":
            with np.errstate(over="ignore"):
                s = np.stack([v[:, a:b].sum(axis=1) for a, b in span], axis=1)
            out[(col, agg)] = (np.where(have, s, 0), have)
        elif agg in ("min", "max"):
            key = np.where(ok, _okey(pt, v.reshape(-1)).reshape(v.shape), np.iinfo(np.int64).max if agg == "min" else np.iinfo(np.int64).min)
            red = np.min if agg == "min" else np.max
            kk = np.stack([red(key[:, a:b], axis=1) for a, b in span], axis=1)
            out[(col, agg)] = (np.where(have, _okey_inv(pt, kk.reshape(-1)).reshape(kk.shape), 0).view(v.dtype), have)
        elif agg == "mean" and pt == cabi.TSKV_PT_F64:
            s = np.stack([panes.column(col, "sum")[0][:, a:b].sum(axis=1) for a, b in span], axis=1)
            out[(col, agg)] = (np.where(have, s / np.maximum(wc, 1), 0), have)
    return out


def assert_folded(got, folded, what):
    for (col, agg), (v, ok) in folded.items():
        g, gok = got.column(col, agg)
        assert (gok == ok).all(), "%s: %s %s validity" % (what, col, agg)
        if v.dtype == np.float64:
            assert np.allclose(g[ok], v[ok], rtol=1e-12, atol=1e-9), "%s: %s %s" % (what, col, agg)
        else:
            assert (g[ok] == v[ok]).all(), "%s: %s %s" % (what, col, agg)


def _pane_query(q, slide, k):
    """The tumbling query of q's panes (every row here is in the floor regime, where origin % slide picks the same panes)."""
    p = make_query(FIELDS, AGGS, width=slide, origin=q.origin, first_bucket_start=q.first_bucket_start + (k - 1) * slide,
                   n_buckets=q.n_buckets - k + 1, group_by_series=q.group_by_series, series_ids=q.series_ids,
                   time_ranges=q.time_ranges, predicates=q.predicates)
    p.columns = q.columns
    return p


def test_page_set_features_against_oracle_panes(engine):
    """group by series, predicates, tombstones, several column groups per series, a host-resident page set with CRC on
    read, overlapping chunks: the sliding scan equals the oracle's tumbling panes folded into windows."""
    rng = np.random.default_rng(21)
    window, slide, origin = 60_000, 20_000, 7_000
    k = n_windows_per_row(window, slide)
    arena, descs, truth = random_arena(rng, n_series=50, n_points=600, fields=FIELDS, null_frac=0.15, jitter=400,
                                       multi_cg=True)
    fbs, nb = sliding_window_grid(1_000_000 - 2_000, 1_000_000 + 2_000_000, window, slide, origin)
    sel = np.array(sorted(rng.choice(np.arange(50), 20, replace=False)), dtype=np.uint32)
    tombs = random_tombstones(rng, descs, 1_000_000, 1_600_000)
    hp = engine.upload_pages(arena, descs, verify_crc=True, host_resident=True)
    dp = engine.upload_pages(arena, descs)
    dp.set_tombstones(tombs)
    for gbs in (False, True):
        for preds in ([], [(1, cabi.TSKV_PT_I64, ">", -20)]):
            q = make_query(FIELDS, AGGS, width=window, origin=origin, first_bucket_start=fbs, n_buckets=nb, group_by_series=gbs,
                           series_ids=sel if gbs else None, predicates=preds, time_ranges=[(1_050_000, 1_700_000)])
            what = "gbs=%s preds=%s" % (gbs, preds)
            panes = orc.scan_aggregate(arena, descs, _pane_query(q, slide, k))
            assert_folded(engine.scan_aggregate(hp, q, slide=slide), fold_panes(panes, k, nb), "host-resident " + what)
            assert_matches_exact(engine.scan_aggregate(hp, q, slide=slide), expand_aggregate(truth, q, slide), what=what)
            panes = orc.scan_aggregate(arena, descs, _pane_query(q, slide, k), tombstones=tombs)
            assert_folded(engine.scan_aggregate(dp, q, slide=slide), fold_panes(panes, k, nb), "tombstones " + what)
    hp.close()
    dp.close()

    arena, descs, files = overlapping_arena(rng, n_series=40)
    pages = engine.upload_pages(arena, descs)
    pages.set_chunk_files(files)
    fbs, nb = sliding_window_grid(1_000_000, 1_000_000 + 2_000_000, window, slide, origin)
    for gbs in (False, True):
        q = make_query(FIELDS, AGGS, width=window, origin=origin, first_bucket_start=fbs, n_buckets=nb, group_by_series=gbs)
        panes = orc.scan_aggregate(arena, descs, _pane_query(q, slide, k), chunk_files=files)
        assert_folded(engine.scan_aggregate(pages, q, slide=slide), fold_panes(panes, k, nb), "overlapping chunks gbs=%s" % gbs)
    pages.close()


def test_two_shard_exchange(engine):
    """Two series shards scanned separately, their exchange regions concatenated like an all-gather and merged: integer
    results bit-exact against row expansion over the whole arena, f64 within its bound."""
    import torch
    from cnosdb_b200.parallel import device_tensor
    window, slide = 50_000, 10_000
    shards = [random_arena(np.random.default_rng(40 + r), n_series=30, n_points=400, fields=FIELDS, null_frac=0.1,
                           jitter=300, ids=range(30 * r, 30 * r + 30)) for r in range(2)]
    truth = {**shards[0][2], **shards[1][2]}
    fbs, nb = sliding_fit_grid(truth, window, slide, 0, [])
    ids = np.arange(60, dtype=np.uint32)
    for gbs in (False, True):
        q = make_query(FIELDS, AGGS, width=window, first_bucket_start=fbs, n_buckets=nb, series_ids=ids, group_by_series=gbs,
                       multi_rank=True)
        exp = expand_aggregate(truth, q, slide)
        scans, regions, keep = [], [], []
        for arena, descs, _ in shards:
            pages = engine.upload_pages(arena, descs)
            s = engine.prepare(pages, q, slide=slide)
            s.run()
            ptr, words = s.exchange_view()
            regions.append(device_tensor(ptr, words, torch.int64, torch.device("cuda", engine.device)).clone())
            scans.append(s)
            keep.append(pages)
        gathered = torch.cat(regions)
        torch.cuda.synchronize()
        for s in scans:
            s.merge_gathered(gathered.data_ptr(), 2)
            # each rank's integer MEAN sum went through f64 before the merge: compare MEAN with the oracle rule there
            assert_matches_exact(s.finalize(), exp, what="2-shard exchange gbs=%s" % gbs, int_mean=False)
            s.close()
        for p in keep:
            p.close()


def test_rows_are_decoded_once_and_graph_replay_is_identical(engine):
    rng = np.random.default_rng(4)
    arena, descs, truth = random_arena(rng, n_series=80, n_points=700, fields=FIELDS, null_frac=0.1, jitter=200)
    pages = engine.upload_pages(arena, descs)
    window, slide = 5 * 60_000, 60_000
    fbs, nb = sliding_window_grid(1_000_000, 1_000_000 + 700_000, window, slide)
    q = make_query(FIELDS, AGGS, width=window, first_bucket_start=fbs, n_buckets=nb, time_ranges=[(1_000_000, 1_700_000)])
    got = engine.scan_aggregate(pages, q, slide=slide)
    c_slide = engine.counters()
    k = n_windows_per_row(window, slide)
    engine.scan_aggregate(pages, _pane_query(q, slide, k))
    c_tumble = engine.counters()
    assert c_slide["points_decoded"] == c_tumble["points_decoded"] > 0
    assert c_slide["page_read_count"] == c_tumble["page_read_count"]
    assert c_slide["rows_in_range"] == c_tumble["rows_in_range"]
    assert_matches_exact(got, expand_aggregate(truth, q, slide))
    s = engine.prepare(pages, q, slide=slide)
    s.run()
    first = s.finalize()
    for _ in range(3):  # the second enqueue captures the pass as a CUDA graph, the later ones replay it
        s.enqueue()
        s.sync()
        _ints_equal(s.finalize(), first, "replayed pass")
    _ints_equal(first, got, "prepared vs one-shot")
    s.close()
    pages.close()
