"""Host-side scan planning heuristics (cnosdb_b200/csrc/host_util.cc), exercised through the host library: the selected
fraction of a shard, the grids of the lane-per-page kernels, the overlap groups of the merge pass and the page parts.
No GPU needed."""
import ctypes as C

import numpy as np

from cnosdb_b200 import cabi
from cnosdb_b200.parallel import select_tag_subset, shard_range


def lib():
    L = cabi.load_hostgen_library()
    L.tskvplan_selected_fraction.argtypes = [C.c_void_p, C.c_uint64, C.c_void_p, C.c_uint64]
    L.tskvplan_selected_fraction.restype = C.c_double
    return L


def frac(arena_ids, sel):
    a = np.ascontiguousarray(arena_ids, dtype=np.uint32)
    if sel is None:
        return lib().tskvplan_selected_fraction(a.ctypes.data, len(a), None, 0)
    s = np.ascontiguousarray(sel, dtype=np.uint32)
    return lib().tskvplan_selected_fraction(a.ctypes.data, len(a), s.ctypes.data, len(s))


def test_selected_fraction_counts_only_ids_inside_the_shard():
    n = 1_000_000
    sel = select_tag_subset(n, 10)  # the global 10 % selection every rank is handed
    for world in (1, 2, 4, 8):
        for rank in (0, world - 1):
            lo, hi = shard_range(n, rank, world)
            f = frac(np.arange(lo, hi), sel)
            assert abs(f - 0.1) < 0.005, (world, rank, f)   # not 0.1 * world
    assert frac(np.arange(100, 200), None) == 1.0
    assert frac(np.arange(100, 200), np.array([5, 7, 300])) == 0.0
    assert frac(np.arange(100, 200), np.arange(0, 1000)) == 1.0


def test_serial_grid_planner_minimises_the_quantised_makespan():
    """plan_serial_grids: a chunk of 32 pages is one serial task, bins finish in whole rounds of their chunk time. For C4
    on one GPU (1250 / 1250 / 313 / 313 chunks, measured chunk times) everything does not fit in one round: the long
    simple8b-timestamp chunks get one round, the RLE bins two; a 1/8 shard fits in a single round."""
    L = lib()
    L.tskvplan_serial_grids.argtypes = [C.c_int, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_void_p]

    def plan(chunks, t, occ, sm=132, wpb=4):
        c = np.array(chunks, dtype=np.float64)
        tt = np.array(t, dtype=np.float64)
        o = np.array(occ, dtype=np.int32)
        g = np.zeros(len(c), dtype=np.int32)
        L.tskvplan_serial_grids(len(c), c.ctypes.data, tt.ctypes.data, o.ctypes.data, sm, wpb, g.ctypes.data)
        return g

    chunks, t, occ = [1250, 1250, 313, 313, 0], [0.28, 0.31, 0.44, 0.47, 1.0], [4, 4, 3, 3, 4]
    g = plan(chunks, t, occ)
    assert g[4] == 0
    rounds = [int(np.ceil(c / (x * 4))) for c, x in zip(chunks[:4], g[:4])]
    assert rounds == [2, 2, 1, 1], (g, rounds)
    assert sum(x / o for x, o in zip(g[:4], occ)) <= 132
    g8 = plan([157, 157, 40, 40], t[:4], occ[:4])
    assert [int(np.ceil(c / (x * 4))) for c, x in zip([157, 157, 40, 40], g8)] == [1, 1, 1, 1]
    # a machine too small even for the largest round count considered still gets a valid (over-subscribed) plan
    g1 = plan([1000], [1.0], [1], sm=2, wpb=4)
    assert g1[0] >= 1


def test_overlap_groups_follow_the_reference_grouping():
    """plan_overlap_groups = build_series_reader's chunk grouping (reader/iterator.rs:463-560): the table of
    reader/utils.rs:330-353 (groups of 4, 2 and 1 chunks), streams ordered by file id, column groups of a chunk in time order."""
    L = lib()
    L.tskvplan_overlap_groups.argtypes = [C.c_uint64] + [C.c_void_p] * 9
    L.tskvplan_overlap_groups.restype = None

    def plan(series, rows, bounds, files):
        n = len(series)
        a = [np.ascontiguousarray(series, dtype=np.uint32), np.ascontiguousarray(rows, dtype=np.uint32),
             np.ascontiguousarray(bounds, dtype=np.int64).reshape(-1, 2), np.ascontiguousarray(files, dtype=np.uint64)]
        merge = np.zeros(n, dtype=np.uint8)
        counts = np.zeros(5, dtype=np.uint64)
        mcg, mst, sgrp = (np.zeros(n, dtype=np.uint32) for _ in range(3))
        L.tskvplan_overlap_groups(n, *[x.ctypes.data for x in a], merge.ctypes.data, counts.ctypes.data, mcg.ctypes.data,
                                  mst.ctypes.data, sgrp.ctypes.data)
        c = [int(x) for x in counts]
        return merge, c, mcg[:c[2]], mst[:c[2]], sgrp[:c[1]]

    trs = [(0, 10), (1, 3), (4, 7), (6, 10), (11, 14), (12, 15), (16, 18)]
    # file ids descending in time order: inside a group the streams must come out ascending by file id
    merge, c, mcg, mst, sgrp = plan([5] * 7, [10] * 7, trs, [70, 60, 50, 40, 30, 20, 10])
    assert merge.tolist() == [1, 1, 1, 1, 1, 1, 0]
    assert c == [2, 6, 6, 60, 3]          # 2 merge groups, 6 streams, 6 merge column groups, 60 rows, 3 overlap groups
    assert mcg.tolist() == [3, 2, 1, 0, 5, 4] and sgrp.tolist() == [0, 0, 0, 0, 1, 1]
    # one file with two column groups (one chunk): never merged with itself; another series' chunks do not interact
    merge, c, mcg, mst, _ = plan([1, 1, 2, 2, 2], [5, 5, 5, 5, 7], [(0, 9), (10, 19), (0, 9), (20, 29), (5, 25)], [1, 1, 1, 1, 2])
    assert merge.tolist() == [0, 0, 1, 1, 1] and c[0] == 1 and c[1] == 2 and c[4] == 2
    assert mcg.tolist() == [2, 3, 4] and mst.tolist() == [0, 0, 1]    # chunk of file 1 = column groups 2, 3 in time order
    # touching ranges overlap (min_ts <= running max), disjoint ones do not
    assert plan([1, 1], [3, 3], [(0, 5), (5, 9)], [1, 2])[0].tolist() == [1, 1]
    assert plan([1, 1], [3, 3], [(0, 5), (6, 9)], [1, 2])[0].tolist() == [0, 0]


def test_page_parts_follow_the_selection_size():
    """Pages cut at restart points: about 4 chunks per resident warp. C4 on one H100 (3 125 chunks of whole pages on
    2 112 warp slots) -> 3 parts of 384 rows; an eighth of it -> one part per 128-row restart interval; C3 (31 k chunks)
    -> whole pages; parts are whole multiples of the interval and never more than the intervals of the longest page."""
    L = lib()
    L.tskvplan_parts_wanted.argtypes = [C.c_double, C.c_double, C.c_double]
    L.tskvplan_parts_wanted.restype = C.c_uint32
    L.tskvplan_bin_parts.argtypes = [C.c_uint32, C.c_uint32, C.c_uint32, C.POINTER(C.c_uint32)]
    L.tskvplan_bin_parts.restype = C.c_uint32

    def bin_parts(maxrows, want, skip=128):
        pr = C.c_uint32(0)
        return L.tskvplan_bin_parts(maxrows, skip, want, C.byref(pr)), pr.value

    warps = 132 * 4 * 4
    assert L.tskvplan_parts_wanted(3125.0, float(warps), 4.0) == 3
    assert L.tskvplan_parts_wanted(391.0, float(warps), 4.0) == 22
    assert bin_parts(1000, 22) == (8, 128)
    assert L.tskvplan_parts_wanted(31250.0, float(warps), 4.0) == 1
    assert L.tskvplan_parts_wanted(0.0, float(warps), 4.0) == 1
    assert bin_parts(1000, 4) == (4, 256)
    assert bin_parts(1000, 25) == (8, 128)
    assert bin_parts(1000, 3) == (3, 384)          # 8 intervals in parts of 3: 3 + 3 + 2
    assert bin_parts(1000, 1) == (1, 0) and bin_parts(128, 8) == (1, 0) and bin_parts(129, 8) == (2, 128)
    assert bin_parts(102_400, 64) == (62, 1664)    # 800 intervals, 13 per part
    for maxrows in (129, 255, 1000, 1024, 1025, 50_000):
        for want in (2, 3, 5, 8, 64, 4096):
            parts, rows = bin_parts(maxrows, want)
            assert rows % 128 == 0 and parts * rows >= maxrows and (parts - 1) * rows < maxrows and parts <= max(want, 1)
