"""GROUP BY tags on the GPU (tskvgpu_*_grouped): a map from selected series slot to group. The main oracle is the scan
itself: group g's cells must equal the ungrouped scan whose series_ids are g's members, for every aggregate including
FIRST / LAST (same tie-break keys). Also checked: the identities (one group == ungrouped, identity map == GROUP BY
series), the exact reference with a group map, sliding windows, the two-shard exchange, graph replay and the refusals."""
import copy
import ctypes as C

import numpy as np
import pytest

from cnosdb_b200 import cabi, datagen
from cnosdb_b200.engine import TskvError, sliding_window_grid
from tests.helpers import (ALL_AGGS, GEOM_AGGS, GEOM_FIELDS, GEOMETRY_CASES, ReferenceError, assert_matches_exact,
                           bucket_spec, exact_fit_grid, geometry_arena, geometry_ranges, make_query,
                           random_arena)
from tests.group_reference import exact_aggregate_grouped
from tests.test_gpu_bool import bool_arena
from tests.test_gpu_overlap_merge import overlapping_arena
from tests.test_gpu_parity import random_tombstones

pytestmark = pytest.mark.gpu

ENVS = ("1", "3")  # TSKV_PARTS
FIELDS = ((1, cabi.TSKV_PT_I64), (2, cabi.TSKV_PT_F64), (3, cabi.TSKV_PT_U64))
AGGS = ("count", "sum", "min", "max", "mean")


def _float_out(res, col, agg):
    return agg == "mean" or (agg == "sum" and res.phys[col] == cabi.TSKV_PT_F64)


def assert_cells_equal(gv, gok, sv, sok, res, col, agg, what, rtol=1e-12):
    """Integer outputs and FIRST / LAST bit for bit; f64 SUM / MEAN (and MEAN) within rtol (summation order)."""
    assert (gok == sok).all(), "%s: %s %s validity" % (what, col, agg)
    if _float_out(res, col, agg):
        assert np.allclose(gv.view(np.float64), sv.view(np.float64), rtol=rtol, atol=1e-9), "%s: %s %s" % (what, col, agg)
    else:
        assert (gv == sv).all(), "%s: %s %s" % (what, col, agg)


def assert_same(a, b, what):
    assert a.names == b.names and a.values.shape == b.values.shape
    for j, (col, agg) in enumerate(a.names):
        assert_cells_equal(a.values[j], a.validity[j], b.values[j], b.validity[j], a, col, agg, what)


def with_series(q, ids):
    s = copy.copy(q)
    s.series_ids = np.ascontiguousarray(ids, dtype=np.uint32)
    s._keep = None
    return s


def assert_groups_match_subsets(engine, pages, q, gmap, n_groups, slot_ids, what, slide=None):
    """Every group's cells of the grouped scan == the ungrouped scan of the group's members; an empty group reads like
    an empty bucket (COUNT 0, every other output NULL)."""
    got = engine.scan_aggregate(pages, q, slide=slide, group_ids=gmap, n_groups=n_groups)
    nb = q.n_buckets
    assert got.n_groups == n_groups and got.values.shape[1] == n_groups * nb
    for g in range(n_groups):
        members = slot_ids[np.asarray(gmap) == g]
        cells = slice(g * nb, (g + 1) * nb)
        if members.size == 0:
            for j, (col, agg) in enumerate(got.names):
                assert (got.values[j][cells] == 0).all(), "%s: empty group %d %s %s" % (what, g, col, agg)
                assert (got.validity[j][cells] == (agg == "count")).all(), "%s: empty group %d %s %s" % (what, g, col, agg)
            continue
        sub = engine.scan_aggregate(pages, with_series(q, members), slide=slide)
        for j, (col, agg) in enumerate(got.names):
            assert_cells_equal(got.values[j][cells], got.validity[j][cells], sub.values[j], sub.validity[j], got, col, agg,
                               "%s group %d (%d series)" % (what, g, members.size))


def make_map(rng, n_slots, n_groups):
    """Random group ids in [0, n_groups): group 0 holds exactly one series and, for n_groups >= 3, the last group none."""
    if n_groups <= 2:
        ids = np.full(n_slots, n_groups - 1, dtype=np.uint32)
    else:
        ids = rng.integers(1, n_groups - 1, n_slots).astype(np.uint32)
    ids[int(rng.integers(0, n_slots))] = 0
    return ids


def _set_env(monkeypatch, parts):
    monkeypatch.setenv("TSKV_PARTS", parts)


def test_identities(engine, monkeypatch):
    """All-zero ids with one group == the ungrouped scan; ids[i] = i with one group per slot == GROUP BY series."""
    rng = np.random.default_rng(3)
    arena, descs, truth = random_arena(rng, n_series=70, n_points=400, fields=FIELDS, null_frac=0.1, multi_cg=True,
                                       raw_frac=0.1)
    pages = engine.upload_pages(arena, descs)
    fbs, nb = bucket_spec(1_000_000, 1_000_000 + 800_000, 30_000, origin=11)
    sel = np.array(sorted(rng.choice(np.arange(70), 40, replace=False)), dtype=np.uint32)
    for ids in (None, sel):
        n = 70 if ids is None else len(ids)
        q = make_query(FIELDS, ALL_AGGS, width=30_000, origin=11, first_bucket_start=fbs, n_buckets=nb, series_ids=ids)
        gbs = make_query(FIELDS, ALL_AGGS, width=30_000, origin=11, first_bucket_start=fbs, n_buckets=nb, series_ids=ids,
                         group_by_series=True)
        for parts in ENVS:
            _set_env(monkeypatch, parts)
            what = "sel=%s parts=%s" % (ids is not None, parts)
            assert_same(engine.scan_aggregate(pages, q, group_ids=np.zeros(n, dtype=np.uint32), n_groups=1),
                        engine.scan_aggregate(pages, q), "one group " + what)
            assert_same(engine.scan_aggregate(pages, q, group_ids=np.arange(n, dtype=np.uint32), n_groups=n),
                        engine.scan_aggregate(pages, gbs), "identity " + what)
    pages.close()


def _arenas(rng):
    """(name, arena, descs, fields, aggs, tombstones or None): equal timestamps across series (ties decide FIRST / LAST),
    nulls, several column groups per series, jittered (simple8b) and raw (generic) pages, boolean pages."""
    a, d, _ = random_arena(rng, n_series=90, n_points=300, fields=FIELDS, null_frac=0.15, multi_cg=True)
    yield "ties", a, d, FIELDS, ALL_AGGS, None
    a, d, _ = random_arena(rng, n_series=90, n_points=300, fields=FIELDS, null_frac=0.1, jitter=400, raw_frac=0.2,
                           multi_cg=True)
    yield "jitter+raw+tombstones", a, d, FIELDS, ALL_AGGS, random_tombstones(rng, d, 1_000_000, 1_250_000)
    a, d = bool_arena(rng, n_series=90)
    yield "bool", a, d, ((1, cabi.TSKV_PT_BOOL), (2, cabi.TSKV_PT_I64)), ("count", "min", "max", "first", "last"), None


def test_subset_equivalence(engine, monkeypatch):
    rng = np.random.default_rng(17)
    for name, arena, descs, fields, aggs, tombs in _arenas(rng):
        pages = engine.upload_pages(arena, descs)
        if tombs is not None:
            pages.set_tombstones(tombs)
        all_ids = np.unique(descs["series_id"]).astype(np.uint32)
        sel = np.array(sorted(rng.choice(all_ids, 60, replace=False)), dtype=np.uint32)
        fbs, nb = bucket_spec(1_000_000 - 1000, 1_000_000 + 1_600_000, 50_000, origin=5)
        preds = [(2, cabi.TSKV_PT_I64, ">", -15)] if name == "bool" else [(1, cabi.TSKV_PT_I64, ">", -20)]
        for ids, pr in ((None, []), (sel, preds)):
            slot_ids = all_ids if ids is None else sel
            q = make_query(fields, aggs, width=50_000, origin=5, first_bucket_start=fbs, n_buckets=nb, series_ids=ids,
                           predicates=pr, time_ranges=[(1_020_000, 1_500_000)])
            for n_groups in (2, 7, 64, len(slot_ids) // 3):
                gmap = make_map(rng, len(slot_ids), n_groups)
                for parts in ENVS:
                    _set_env(monkeypatch, parts)
                    assert_groups_match_subsets(engine, pages, q, gmap, n_groups, slot_ids, "%s sel=%s G=%d parts=%s" % (
                        name, ids is not None, n_groups, parts))
        pages.close()


@pytest.mark.parametrize("case", GEOMETRY_CASES[::5], ids=[c[0] for c in GEOMETRY_CASES[::5]])
def test_exact_reference_geometry(engine, case, monkeypatch):
    """COUNT / SUM / MIN / MAX / MEAN against the exact reference with a group map, in two layouts: one group per block of
    40 series (whole warps of identical RLE pages share a group: the uniform schedule runs) and groups interleaved slot by
    slot (every warp holds many groups: the vote falls back)."""
    name, step, w, origin, t0, n, kinds = case
    arena, descs, truth = geometry_arena(len(name), t0, step, n)
    pages = engine.upload_pages(arena, descs)
    slots = np.arange(len(truth))
    layouts = [("blocks", (slots // 40).astype(np.uint32), 3), ("interleaved", (slots % 60).astype(np.uint32), 60)]
    for kind in kinds[:2]:
        ranges = geometry_ranges(kind, t0, step, n, w, origin)
        fbs, nb = exact_fit_grid(truth, w, origin, ranges)
        q = make_query(GEOM_FIELDS, GEOM_AGGS, width=w, origin=origin, first_bucket_start=fbs, n_buckets=nb, time_ranges=ranges)
        for lname, gmap, n_groups in layouts:
            if n_groups * nb > 300_000:
                continue
            try:
                exp, err = exact_aggregate_grouped(truth, q, gmap, n_groups), None
            except ReferenceError as e:
                exp, err = None, e.status
            for parts in ENVS:
                _set_env(monkeypatch, parts)
                what = "%s %s %s parts=%s" % (name, kind, lname, parts)
                try:
                    got, st = engine.scan_aggregate(pages, q, group_ids=gmap, n_groups=n_groups), None
                except TskvError as e:
                    got, st = None, e.status
                assert st == err, "%s: status %s, expected %s" % (what, st, err)
                if err is None:
                    assert_matches_exact(got, exp, what=what)
    pages.close()


def test_other_paths(engine, monkeypatch):
    """Overlapping chunks (the merge pass), a host-resident page set, the item-driven work list and a table too large for
    shared memory: each grouped scan against the subset scans of the same configuration."""
    rng = np.random.default_rng(23)
    fbs, nb = bucket_spec(1_000_000, 1_000_000 + 3_000_000, 60_000)
    arena, descs, files = overlapping_arena(rng, n_series=50)
    pages = engine.upload_pages(arena, descs)
    pages.set_chunk_files(files)
    all_ids = np.unique(descs["series_id"]).astype(np.uint32)
    q = make_query(FIELDS, ALL_AGGS, width=60_000, first_bucket_start=fbs, n_buckets=nb)
    for n_groups in (2, 7):
        assert_groups_match_subsets(engine, pages, q, make_map(rng, len(all_ids), n_groups), n_groups, all_ids,
                                    "overlapping chunks G=%d" % n_groups)
    pages.close()

    arena, descs, _ = random_arena(rng, n_series=80, n_points=500, fields=FIELDS, null_frac=0.1, jitter=300, multi_cg=True)
    all_ids = np.arange(80, dtype=np.uint32)
    hp = engine.upload_pages(arena, descs, verify_crc=True, host_resident=True)
    dp = engine.upload_pages(arena, descs)
    fbs, nb = bucket_spec(1_000_000 - 300, 1_000_000 + 1_000_000, 20_000)
    for aggs in (AGGS, ALL_AGGS):
        q = make_query(FIELDS, aggs, width=20_000, first_bucket_start=fbs, n_buckets=nb)
        gmap = make_map(rng, 80, 7)
        assert_groups_match_subsets(engine, hp, q, gmap, 7, all_ids, "host-resident %s" % (aggs,))
        for env, val in (("TSKV_WORKLIST", "items"), ("TSKV_SMEM_TABLE_KB", "0")):
            with monkeypatch.context() as m:
                m.setenv(env, val)
                for parts in ENVS:
                    _set_env(m, parts)
                    assert_groups_match_subsets(engine, dp, q, gmap, 7, all_ids, "%s=%s %s parts=%s" % (env, val, aggs, parts))
    hp.close()
    dp.close()


def test_sliding_windows(engine, monkeypatch):
    rng = np.random.default_rng(29)
    arena, descs, _ = random_arena(rng, n_series=60, n_points=500, fields=FIELDS, null_frac=0.1, jitter=200, multi_cg=True)
    pages = engine.upload_pages(arena, descs)
    window, slide = 60_000, 20_000
    fbs, nb = sliding_window_grid(1_000_000 - 2_000, 1_000_000 + 1_200_000, window, slide)
    q = make_query(FIELDS, AGGS, width=window, first_bucket_start=fbs, n_buckets=nb, predicates=[(1, cabi.TSKV_PT_I64, ">", -30)])
    ids = np.arange(60, dtype=np.uint32)
    for n_groups in (2, 7, 20):
        gmap = make_map(rng, 60, n_groups)
        for parts in ENVS:
            _set_env(monkeypatch, parts)
            assert_groups_match_subsets(engine, pages, q, gmap, n_groups, ids, "sliding G=%d parts=%s" % (n_groups, parts),
                                        slide=slide)
    # slide == window: the tumbling grouped scan
    fbs, nb = bucket_spec(1_000_000 - 2_000, 1_000_000 + 1_200_000, window)
    q = make_query(FIELDS, ALL_AGGS, width=window, first_bucket_start=fbs, n_buckets=nb)
    assert_same(engine.scan_aggregate(pages, q, slide=window, group_ids=gmap, n_groups=20),
                engine.scan_aggregate(pages, q, group_ids=gmap, n_groups=20), "slide == window")
    pages.close()


def _arena_from_truth(truth, fields):
    b = datagen.ArenaBuilder()
    for sid in sorted(truth):
        for ts, cols in truth[sid]:
            b.add_column_group(sid, ts, [(c, pt, cols[c][0], None if cols[c][1].all() else cols[c][1]) for c, pt in fields])
    return b.finish()


def test_two_shard_exchange(engine):
    """Two series shards scanned separately with the global series_ids and group map, exchange regions concatenated like
    an all-gather and merged: equal to the grouped scan of one page set holding both shards."""
    import torch
    from cnosdb_b200.parallel import device_tensor
    shards = [random_arena(np.random.default_rng(60 + r), n_series=30, n_points=400, fields=FIELDS, null_frac=0.1,
                           jitter=300, ids=range(30 * r, 30 * r + 30)) for r in range(2)]
    truth = {**shards[0][2], **shards[1][2]}
    whole = engine.upload_pages(*_arena_from_truth(truth, FIELDS))
    ids = np.arange(60, dtype=np.uint32)
    gmap = make_map(np.random.default_rng(61), 60, 7)
    fbs, nb = bucket_spec(1_000_000 - 300, 1_000_000 + 400_000, 25_000)
    for window, slide, aggs in ((25_000, None, ALL_AGGS), (50_000, 25_000, AGGS)):
        fb, n = (fbs, nb) if slide is None else sliding_window_grid(1_000_000 - 300, 1_000_000 + 400_000, window, slide)
        q = make_query(FIELDS, aggs, width=window, first_bucket_start=fb, n_buckets=n, series_ids=ids, multi_rank=True)
        exp = engine.scan_aggregate(whole, q, slide=slide, group_ids=gmap, n_groups=7)
        scans, regions, keep = [], [], []
        for arena, descs, _ in shards:
            pages = engine.upload_pages(arena, descs)
            s = engine.prepare(pages, q, slide=slide, group_ids=gmap, n_groups=7)
            s.run()
            ptr, words = s.exchange_view()
            regions.append(device_tensor(ptr, words, torch.int64, torch.device("cuda", engine.device)).clone())
            scans.append(s)
            keep.append(pages)
        gathered = torch.cat(regions)
        torch.cuda.synchronize()
        for s in scans:
            s.merge_gathered(gathered.data_ptr(), 2)
            assert_same(s.finalize(), exp, "2-shard exchange slide=%s" % slide)
            s.close()
        for p in keep:
            p.close()
    whole.close()


def test_graph_replay(engine):
    rng = np.random.default_rng(31)
    arena, descs, _ = random_arena(rng, n_series=80, n_points=600, fields=FIELDS, null_frac=0.1, jitter=200)
    pages = engine.upload_pages(arena, descs)
    fbs, nb = bucket_spec(1_000_000 - 200, 1_000_000 + 600_000, 30_000)
    gmap = make_map(rng, 80, 9)
    for aggs in (AGGS, ALL_AGGS):
        q = make_query(FIELDS, aggs, width=30_000, first_bucket_start=fbs, n_buckets=nb)
        once = engine.scan_aggregate(pages, q, group_ids=gmap, n_groups=9)
        s = engine.prepare(pages, q, group_ids=gmap, n_groups=9)
        for _ in range(3):  # the second enqueue captures the pass as a CUDA graph, the third replays it
            s.enqueue()
            s.sync()
        assert_same(s.finalize(), once, "graph replay %s" % (aggs,))
        s.close()
    pages.close()


def test_refusals(engine):
    rng = np.random.default_rng(37)
    arena, descs, _ = random_arena(rng, n_series=8, n_points=100, fields=FIELDS)
    pages = engine.upload_pages(arena, descs)
    fbs, nb = bucket_spec(1_000_000, 1_000_000 + 100_000, 10_000)
    base = dict(width=10_000, first_bucket_start=fbs, n_buckets=nb)
    q = make_query(FIELDS, AGGS, **base)
    ok = np.zeros(8, dtype=np.uint32)
    invalid = [
        (q, None, 3, None),                                               # group_ids == NULL
        (q, ok, 0, None),                                                 # n_groups == 0
        (q, np.array([0, 1, 2, 3, 0, 0, 0, 4], dtype=np.uint32), 4, None),  # an id >= n_groups
        (make_query(FIELDS, AGGS, group_by_series=True, **base), ok, 1, None),
        (make_query(FIELDS, AGGS, **dict(base, n_buckets=2)), ok, 2**31, None),  # 2^32 cells
        (make_query(FIELDS, ("count", "first"), multi_rank=True, **base), ok, 1, None),  # multi-rank without series_ids
        (q, ok, 1, -5),                                                   # slide < 0
    ]
    for k, (qq, gmap, n_groups, slide) in enumerate(invalid):
        for call in (engine.scan_aggregate, engine.prepare):
            with pytest.raises(TskvError) as e:
                call(pages, qq, slide=slide, group_ids=gmap, n_groups=n_groups)
            assert e.value.status == cabi.TSKV_ERR_INVALID_ARG, (k, call)
        # the scan itself refuses too, not only the layout
        raw, h = qq.to_c(), C.c_void_p()
        gp = None if gmap is None else np.ascontiguousarray(gmap).ctypes.data
        if k < 5:  # (the layout knows neither multi-rank nor the slide)
            assert engine.lib.tskvgpu_query_output_layout_grouped(pages.handle, C.byref(raw), gp, n_groups,
                                                                  C.byref(cabi.OutputLayout())) == cabi.TSKV_ERR_INVALID_ARG, k
        assert engine.lib.tskvgpu_scan_prepare_grouped(engine.ctx, pages.handle, C.byref(raw), gp, n_groups, slide or 0,
                                                       C.byref(h)) == cabi.TSKV_ERR_INVALID_ARG, k
        assert not h.value
    # grouped sliding windows keep the sliding refusals: FIRST / LAST
    fb, n = sliding_window_grid(1_000_000, 1_000_000 + 100_000, 10_000, 2_000)
    qs = make_query(FIELDS, ("count", "last"), width=10_000, first_bucket_start=fb, n_buckets=n)
    with pytest.raises(TskvError) as e:
        engine.scan_aggregate(pages, qs, slide=2_000, group_ids=ok, n_groups=1)
    assert e.value.status == cabi.TSKV_ERR_UNSUPPORTED
    pages.close()
