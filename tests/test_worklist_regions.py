"""The work list's series-id lookup and bucket regions: the planners on the CPU (which id spaces get the direct id -> rank
table, where each (bin, column, narrow flag) bucket's region starts), and scans whose selections look ids up through the
table, through the binary search, outside the page set's id range and between its ids, against the CPU oracle; and the
work list itself, read back after a pass (tskvgpu_scan_work_list): every chunk of 32 items holds one (bin, column,
narrow flag) bucket and the buckets hold exactly the selected field pages, with GROUP BY tags, a split walk, time
pruning and a host-resident page set."""
import ctypes as C

import numpy as np
import pytest

from cnosdb_b200 import cabi, datagen
from cnosdb_b200.engine import PushedAggregate, QueryOption
from oracle import pyoracle as orc
from tests.helpers import assert_results_equal, bucket_spec

SLACK = 16384  # SERIES_MAP_SLACK (host_util.h)


def lib():
    L = cabi.load_hostgen_library()
    L.tskvplan_series_map.argtypes = [C.c_uint32, C.c_uint32, C.c_uint64]
    L.tskvplan_series_map.restype = C.c_int
    L.tskvplan_worklist_regions.argtypes = [C.c_uint32, C.c_void_p, C.c_void_p]
    L.tskvplan_worklist_regions.restype = C.c_int
    return L


def regions(capacity):
    cap = np.ascontiguousarray(capacity, dtype=np.uint32)
    start = np.zeros(len(cap) + 1, dtype=np.uint32)
    ok = lib().tskvplan_worklist_regions(len(cap), cap.ctypes.data, start.ctypes.data)
    return bool(ok), start


def test_series_map_only_for_dense_id_spaces():
    L = lib()
    assert L.tskvplan_series_map(0, 999_999, 1_000_000)             # one contiguous shard
    assert L.tskvplan_series_map(500_000, 999_999, 500_000)
    assert L.tskvplan_series_map(0, 2 * 1000 - 2, 1000)              # every other id
    assert L.tskvplan_series_map(7, 7, 1)
    assert L.tskvplan_series_map(0, 2 * 10 + SLACK - 1, 10)          # span 2 n + slack
    assert not L.tskvplan_series_map(0, 2 * 10 + SLACK, 10)
    assert not L.tskvplan_series_map(0, 2**32 - 1, 1000)             # ids spread over the whole 32-bit space
    assert not L.tskvplan_series_map(0, 0, 0)                        # no series


def test_worklist_regions_start_on_chunk_boundaries_and_hold_their_capacity():
    rng = np.random.default_rng(5)
    for n in (1, 2, 26, 260):
        cap = rng.integers(0, 200, n).astype(np.uint32)
        cap[rng.random(n) < 0.3] = 0
        ok, start = regions(cap)
        assert ok
        assert start[0] == 0
        assert (start % 32 == 0).all()
        size = np.diff(start.astype(np.int64))
        assert (size >= cap).all() and (size < cap.astype(np.int64) + 32).all()
        assert (size[cap == 0] == 0).all()
    ok, start = regions([])
    assert ok and start.tolist() == [0]
    ok, start = regions([33, 0, 32, 1])
    assert start.tolist() == [0, 64, 64, 96, 128]


def test_worklist_regions_refuse_lists_beyond_32_bit_indices():
    ok, _ = regions([2**31, 2**31])
    assert not ok
    ok, start = regions([2**31, 2**31 - 64])
    assert ok and start[-1] == 2**32 - 64


def _scan_against_oracle(engine, g, sel, what):
    w = 60_000_000_000
    fbs, nb = bucket_spec(datagen.TSBS_T0 - 1_000_000, datagen.TSBS_T0 + 299 * datagen.TSBS_STEP + 1_000_000, w)
    aggs = ["count", "sum", "min", "max", "mean"]
    q = QueryOption([PushedAggregate(1, cabi.TSKV_PT_I64, aggs), PushedAggregate(3, cabi.TSKV_PT_F64, aggs)],
                    series_ids=np.unique(np.asarray(sel, dtype=np.uint32)), width=w, first_bucket_start=fbs, n_buckets=nb)
    pages = engine.upload_pages(g.arena, g.descs)
    try:
        got = engine.scan_aggregate(pages, q)
        c = engine.counters()
    finally:
        pages.close()
    exp = orc.scan_aggregate(g.arena, g.descs, q, n_threads=4)
    assert_results_equal(got, exp, what=what)
    return c


@pytest.mark.gpu
@pytest.mark.parametrize("first, stride", [(0, 1), (1000, 2), (5, 100), (4_000_000_000, 7)])
def test_selection_lookup(engine, first, stride):
    """Dense ids (table), ids with holes (table entries without series), sparse ids (binary search), and ids near the
    top of the 32-bit space; selections mix held ids, ids between them and ids outside [min id, max id]."""
    n = 600
    g = datagen.generate(n, n_fields=2, n_points=300, value_kind=datagen.MIXED, seed=11, first_series_id=first,
                         series_stride=stride, jitter_permille=200, jitter_max=999_999)
    ids = first + stride * np.arange(n, dtype=np.int64)
    held = ids[::3]
    between = (ids[1::5] + 1) if stride > 1 else np.array([], dtype=np.int64)
    outside = np.array([max(first - 1, 0) if first else 0, ids[-1] + 1, ids[-1] + 12345, 2**32 - 1], dtype=np.int64)
    outside = outside[(outside < first) | (outside > ids[-1])]
    try:
        c = _scan_against_oracle(engine, g, np.concatenate([held, between, outside]), "first %d stride %d" % (first, stride))
        assert c["page_read_count"] == 2 * len(held)          # the time page + the queried field page of a held series
        c = _scan_against_oracle(engine, g, np.concatenate([between, outside]), "no held id")
        assert c["page_read_count"] == 0
    finally:
        g.close()


def _regions_arena(rng):
    """300 series of one column group + one series of 80 (its walk is split over several threads). Short (<= 1024 rows)
    and long pages, regular (RLE) and jittered (simple8b) timestamps, narrow and wide i64 values in the same bins, a
    u64 column some groups lack; column group g covers its own stretch of time, so time ranges prune whole groups."""
    b = datagen.ArenaBuilder()
    bounds = []
    groups = [(sid, 1) for sid in range(300)] + [(1000, 80)]
    g = 0
    for sid, n_cg in groups:
        for _ in range(n_cg):
            n = int(rng.choice([200, 900, 1500, 3000]))
            t0 = 10**9 + g * 10**7
            step = np.full(n, 1000, dtype=np.int64)
            if g % 2:
                step += rng.integers(0, 50, n)
            ts = t0 + np.cumsum(step)
            iv = np.cumsum(rng.integers(-5, 6, n))
            if g % 3 == 0:
                iv = iv + 10**15                                  # wide: outside 32 bits
            fields = [(1, cabi.TSKV_PT_I64, iv, None), (2, cabi.TSKV_PT_F64, rng.normal(size=n), None)]
            if g % 4:
                fields.append((3, cabi.TSKV_PT_U64, rng.integers(0, 1000, n).astype(np.uint64), None))
            b.add_column_group(sid, ts, fields)
            bounds.append((int(ts[0]), int(ts[-1])))
            g += 1
    arena, descs = b.finish()
    return arena, descs, np.array(bounds, dtype=np.int64)


def _check_work_list(wl, descs, cols, slot_of, cg_in_time):
    n_cols = len(cols)
    start, fill = wl["region_start"].astype(np.int64), wl["fill"].astype(np.int64)
    n_buckets = len(fill)
    assert n_buckets % (2 * n_cols) == 0
    assert (start % 32 == 0).all() and (fill <= np.diff(start)).all()
    is_time = descs["phys_type"] == cabi.TSKV_PT_TIME
    cg_of = np.cumsum(is_time) - 1                                # column group of every descriptor
    time_page = np.flatnonzero(is_time)[cg_of]
    page, qcol, slot = wl["work_page"], wl["work_qcol"], wl["work_slot"]
    placed = []
    for k in range(n_buckets):
        b, c, f = k // (2 * n_cols), (k // 2) % n_cols, k % 2
        w = np.arange(start[k], start[k] + fill[k])
        p = page[w].astype(np.int64)
        assert (wl["page_bin"][p] == b).all() and ((qcol[w] & 0x7F) == c).all(), k
        assert (descs["column_id"][p] == cols[c]).all() and (wl["page_narrow"][p] == f).all(), k
        # the fused kernel's chunks of the bucket: 32 items from the region start on, never past the fill
        for g0 in range(start[k], start[k] + fill[k], 32):
            chunk = page[g0:min(g0 + 32, start[k] + fill[k])].astype(np.int64)
            keys = {(int(wl["page_bin"][q]), int(descs["column_id"][q]), int(wl["page_narrow"][q])) for q in chunk}
            assert len(keys) == 1, (k, g0, keys)
        assert (slot[w] == [slot_of[int(sid)] for sid in descs["series_id"][p]]).all(), k
        placed.append(w)
    placed = np.concatenate(placed)
    p = page[placed].astype(np.int64)
    expected = np.flatnonzero(~is_time & np.isin(descs["column_id"], cols) & np.isin(descs["series_id"], list(slot_of))
                              & cg_in_time[cg_of])
    assert np.array_equal(np.sort(p), expected)                   # every selected field page once, nothing else
    # one item of every (column group, bin) brings the group's time page
    with_time = (qcol[placed] & 0x80) != 0
    key = cg_of[p] * 64 + wl["page_bin"][p]
    assert np.array_equal(np.unique(key[with_time], return_counts=True)[0], np.unique(key))
    assert (np.unique(key[with_time], return_counts=True)[1] == 1).all()
    return p


@pytest.mark.gpu
@pytest.mark.parametrize("case", ["selection", "tags", "pruned", "host"])
def test_chunks_hold_one_bucket_and_buckets_hold_the_selected_pages(engine, case):
    rng = np.random.default_rng(17)
    arena, descs, bounds = _regions_arena(rng)
    cols = [1, 2, 3]
    sel = np.concatenate([np.arange(0, 300, 2), [1000]]).astype(np.uint32)
    ranges = []
    cg_in_time = np.ones(len(bounds), dtype=bool)
    if case == "pruned":
        ranges = [(10**9 + 40 * 10**7, 10**9 + 200 * 10**7), (10**9 + 330 * 10**7, 10**9 + 350 * 10**7)]
        cg_in_time = np.zeros(len(bounds), dtype=bool)
        for lo, hi in ranges:
            cg_in_time |= (bounds[:, 0] <= hi) & (bounds[:, 1] >= lo)
    q = QueryOption([PushedAggregate(1, cabi.TSKV_PT_I64, ["count", "sum", "min", "max"]),
                     PushedAggregate(2, cabi.TSKV_PT_F64, ["count", "sum"]),
                     PushedAggregate(3, cabi.TSKV_PT_U64, ["count", "max"])],
                    series_ids=sel, time_ranges=ranges)
    groups = (np.arange(len(sel)) * 7 % 5).astype(np.uint32) if case == "tags" else None
    pages = engine.upload_pages(arena, descs, host_resident=case == "host")
    scan = engine.prepare(pages, q, group_ids=groups)
    try:
        scan.run()
        wl = scan.work_list()
    finally:
        scan.close()
        pages.close()
    slot_of = {int(s): i for i, s in enumerate(sel)}
    p = _check_work_list(wl, descs, cols, slot_of, cg_in_time)
    assert len(p) > 200
    L = lib()
    L.tskvplan_walk_split.argtypes = [C.c_uint32, C.c_uint64, C.c_uint64, C.c_uint32]
    L.tskvplan_walk_split.restype = C.c_uint32
    n_field_pages = int((descs["phys_type"] != cabi.TSKV_PT_TIME).sum())
    assert L.tskvplan_walk_split(80, len(sel), n_field_pages, 256) > 1     # the 80-group series is walked by S > 1 threads
    if case == "host":
        assert not wl["page_narrow"].any()                        # host-resident page sets have no narrow flags
    else:
        narrow = wl["page_narrow"][p].astype(bool)
        assert narrow.any() and (~narrow).any()
        bins = wl["page_bin"][p]
        assert set(bins[narrow]) & set(bins[~narrow])             # some bin holds both kinds: its buckets are split
