"""The pair and median references over overlapping chunk files and the random operand cases, with no GPU code:
covariance_reference.paired_rows with `files=` against the hand-merged truth of tests/exact_arenas.two_file_arena (the
arena of the overlap tests of tests/test_gpu_covariance.py and tests/test_gpu_median.py), and on the random operand
cases of tests/sweep_reference.py the pair (c, c)'s n and the median's validity against COUNT(c) of the independent
exact reference, in every cell."""
import copy

import numpy as np
import pytest

from cnosdb_b200 import cabi
from cnosdb_b200.engine import PushedAggregate, QueryOption
from tests import sweep_reference as sw
from tests import test_increase_kernel_list as increase_kernels
from tests import test_median_kernel_list as median_kernels
from tests import test_pair_kernel_list as pair_kernels
from tests.covariance_reference import exact_pair_cells, paired_rows
from tests.exact_arenas import two_file_arena
from tests.helpers import bucket_spec
from tests.increase_reference import exact_increase_cells
from tests.median_reference import exact_median_cells

I64, F64 = cabi.TSKV_PT_I64, cabi.TSKV_PT_F64
T0, STEP, W = 1_000_000, 1000, 50_000
BASE_SEED = 20261017  # tests/test_gpu_kernel_sweep.py's
N_CASES = 60


def test_paired_rows_with_files_match_the_hand_merged_truth():
    _, _, truth, files, merged = two_file_arena(T0, STEP)
    fbs, nb = bucket_spec(T0 - 10 * STEP, T0 + 200 * STEP, W)
    for gbs in (True, False):
        q = QueryOption([], first_bucket_start=fbs, n_buckets=nb, width=W, group_by_series=gbs)
        for pair in ((1, I64, 2, F64), (2, F64, 1, I64), (1, I64, 1, I64)):
            got = paired_rows(truth, q, pair, files=files)
            assert got == paired_rows(merged, q, pair), (gbs, pair)
            assert sum(len(x) for x, _ in got.values()) > 0
        for col, pt in ((1, I64), (2, F64)):
            a = exact_median_cells(truth, q, col, pt, 6 * nb, files=files)
            b = exact_median_cells(merged, q, col, pt, 6 * nb)
            np.testing.assert_array_equal(a[1], b[1])
            np.testing.assert_array_equal(a[0], b[0])
    # without files the same arena holds every row of both files: the merge does change the result
    q = QueryOption([], first_bucket_start=fbs, n_buckets=nb, width=W, group_by_series=True)
    assert paired_rows(truth, q, (1, I64, 2, F64)) != paired_rows(merged, q, (1, I64, 2, F64))


def test_paired_rows_with_files_predicates_and_tombstones():
    """Predicates act on the chunks before the merge: a predicate that only file 2's row fails lets file 1's value of a
    shared time through. A row drop removes a series' times from both files, and a column tombstone masks one
    operand of the merged rows; both against the hand-merged truth."""
    _, _, truth, files, _ = two_file_arena(T0, STEP)
    q = QueryOption([], n_buckets=1, predicates=[(2, F64, ">=", 5.0)])
    got = paired_rows(truth, q, (1, I64, 1, I64), files=files)
    want = []
    for sid in sorted(truth):
        by_t = {}
        for ts, cols in truth[sid]:  # (file 1, then file 2: the later file's row comes last)
            x, xv = cols[1]
            y, yv = cols[2]
            for i, t in enumerate(ts.tolist()):
                if yv[i] and y[i] >= 5.0 and xv[i]:
                    by_t[t] = float(x[i])
        want += [by_t[t] for t in sorted(by_t)]
    assert sorted(got[0][0]) == sorted(want)
    _, _, _, _, merged = two_file_arena(T0, STEP)
    masked, dropped = (T0 + 60 * STEP, T0 + 80 * STEP), (T0, T0 + 100 * STEP)
    tombs = cabi.tombstones([(0, 1, *masked), (1, None, *dropped)])
    q = QueryOption([], n_buckets=1, group_by_series=True)
    for pair in ((1, I64, 2, F64), (2, F64, 1, I64)):
        got = paired_rows(truth, q, pair, tombstones=tombs, files=files)
        want = {}
        for sid, [(ts, cols)] in merged.items():
            (x, xv), (y, yv) = cols[pair[0]], cols[pair[2]]
            for i, t in enumerate(ts.tolist()):
                if not (xv[i] and yv[i]) or (sid == 0 and masked[0] <= t <= masked[1]) or \
                        (sid == 1 and dropped[0] <= t <= dropped[1]):
                    continue
                xs, ys = want.setdefault(sid, ([], []))
                xs.append(float(x[i]))
                ys.append(float(y[i]))
        assert got == want, pair
        assert len(got[1][0]) < len(paired_rows(merged, q, pair)[1][0])  # (the tombstones do drop rows)


def count_result(case, col):
    """COUNT(col) of the case's query (its selection, grouping, tombstones and files) by the exact reference of the
    fused scan, or None when that reference refuses the case."""
    q = copy.copy(case.query)
    q.columns, q.pairs, q._keep = [PushedAggregate(col, sw.COLUMNS[col], ["count"])], [], None
    res = sw.expected(case.truth, q, case.extra, tombstones=case.tombstones, files=case.files)
    return None if isinstance(res, (int, str)) else res.values[0]


@pytest.mark.parametrize("index", range(N_CASES))
def test_pair_n_and_median_validity_are_count(index):
    """The pair (c, c) counts exactly the rows COUNT(c) counts, and the median of c is valid exactly where
    COUNT(c) > 0, in every cell, for every numeric column of a random operand case."""
    case = sw.random_operand_case(index, BASE_SEED)
    if "slide" in case.extra:
        return
    kw = dict(tombstones=case.tombstones, files=case.files, group_ids=case.extra.get("group_ids"),
              edges=case.extra.get("edges"), labels=case.extra.get("labels"))
    for col in sw.columns_of(case.truth):
        pt = sw.COLUMNS[col]
        if pt == sw.BOOL:
            continue
        count = count_result(case, col)
        if count is None:
            return
        n, _, _, _ = exact_pair_cells(case.truth, case.query, (col, pt, col, pt), count.size, **kw)
        np.testing.assert_array_equal(n, count, err_msg="%s column %d" % (case.describe(), col))
        _, ok = exact_median_cells(case.truth, case.query, col, pt, count.size, **kw)
        np.testing.assert_array_equal(ok, count > 0, err_msg="%s column %d" % (case.describe(), col))


def test_operand_cases_cover_the_features():
    """The random operand cases hold pairs with x == y and mixed types, two medians on one column, medians on projected
    and unprojected columns, files, and every operand refusal."""
    seen = set()
    for i in range(200):
        case = sw.random_operand_case(i, BASE_SEED)
        q = case.query
        seen.add("refusal " + case.desc["operand_refusal"])
        for x, xt, y, yt in q.pairs:
            seen.add("x == y" if x == y else "x != y")
            seen.add("mixed types" if xt != yt else "one type")
        meds = [c.column_id for c in q.columns if c.median]
        if len(meds) > len(set(meds)):
            seen.add("two medians on one column")
        for c in q.columns:
            if c.median:
                seen.add("projected median" if c.agg_mask or c.column_id in [p.column_id for p in q.projected()]
                         else "unprojected median")
        if (q.pairs or meds) and case.files is not None:
            seen.add("files")
    want = {"refusal none", "refusal pair_sliding", "refusal median_sliding", "refusal bool_pair",
            "refusal bool_median", "x == y", "x != y", "mixed types", "two medians on one column", "projected median",
            "unprojected median", "files"}
    assert want <= seen, want - seen


def test_operand_kernels_are_the_librarys():
    """sweep_reference.OPERAND_KERNELS is exactly the scan and merged-row subset of the pair, median and increase
    kernels the kernel-list tests hold to the library."""
    both = pair_kernels.EXPECTED | median_kernels.EXPECTED | increase_kernels.EXPECTED
    prefixes = ("k_scan_pair<", "k_merge_pairs_rows<", "k_scan_median<", "k_merge_median_rows", "k_scan_increase<",
                "k_merge_increase")
    want = {k for k in both if k.startswith(prefixes)}
    assert set(sw.OPERAND_KERNELS) == want and len(sw.OPERAND_KERNELS) == len(want)


def test_first_cases_unchanged_by_the_operand_draw():
    """random_operand_case and random_increase_case draw their operands from streams of their own: the case underneath
    is random_case's (its arena and every draw), and random_operand_case's cases do not change."""
    for i in range(20):
        a, b, c = sw.random_case(i, BASE_SEED), sw.random_operand_case(i, BASE_SEED), sw.random_increase_case(i, BASE_SEED)
        assert {k: b.desc[k] for k in a.desc} == a.desc, i
        assert {k: c.desc[k] for k in a.desc} == a.desc, i
        assert (c.arena == a.arena).all() and (c.descs == a.descs).all(), i
        assert not any(x.increase for x in b.query.columns), i


N_INC_CASES = 150  # tests/test_gpu_kernel_sweep.py's N_INCREASE


def test_increase_cases_cover_the_shapes_and_refusals():
    """The random increase cases hold every accepted shape, kept groupings that are accepted and refused, every
    refusal of increase_status, duplicates, unprojected operands, a pair or a median beside increases, and files."""
    seen = set()
    for i in range(N_INC_CASES):
        case = sw.random_increase_case(i, BASE_SEED)
        q = case.query
        incs = [c.column_id for c in q.columns if c.increase]
        if not incs:
            continue
        exp = sw.increase_status(case.truth, q, case.extra)
        seen.add("%s %s" % (case.desc["shape"], "accepted" if exp is None else "refused"))
        if exp is not None:
            seen.add("refusal %s" % exp)
            if exp == cabi.TSKV_ERR_UNSUPPORTED:
                seen.add("unsupported: " + ("labels" if "labels" in case.extra else "tags" if "group_ids" in case.extra
                                            else "ungrouped"))
        if len(incs) > len(set(incs)):
            seen.add("duplicate")
        if any(c not in [p.column_id for p in q.projected()] for c in incs):
            seen.add("unprojected")
        if q.pairs or any(c.median for c in q.columns):
            seen.add("pair or median")
        if case.files is not None and exp is None:
            seen.add("files")
    want = {"series accepted", "tags accepted", "edges accepted", "one accepted", "kept accepted", "kept refused",
            "refusal ValueError", "refusal %d" % cabi.TSKV_ERR_INVALID_ARG, "refusal %d" % cabi.TSKV_ERR_UNSUPPORTED,
            "unsupported: labels", "unsupported: tags", "unsupported: ungrouped", "duplicate", "unprojected",
            "pair or median", "files"}
    assert want <= seen, want - seen


def test_increase_status_order():
    """increase_status gives the first refusal in the library's order when several apply: the engine's ValueError for a
    sliding window, then a BOOL operand, then labels, a shared tag group, an ungrouped scan over several series."""
    truth = {0: [], 1: []}
    inc = lambda c, pt: PushedAggregate(c, pt, ["increase"])  # noqa: E731
    q = QueryOption([inc(4, sw.BOOL)])
    lab = {"edges": np.array([0, 5, 9]), "labels": np.zeros(2, dtype=np.uint32)}
    assert sw.increase_status(truth, q, dict(lab, slide=5)) == "ValueError"
    assert sw.increase_status(truth, q, lab) == cabi.TSKV_ERR_INVALID_ARG
    q = QueryOption([inc(1, I64)])
    assert sw.increase_status(truth, q, dict(lab, group_ids=np.zeros(2, dtype=np.uint32))) == cabi.TSKV_ERR_UNSUPPORTED
    assert sw.increase_status(truth, q, {"group_ids": np.array([1, 0], dtype=np.uint32)}) is None
    assert sw.increase_status(truth, q, {"group_ids": np.array([1, 1], dtype=np.uint32)}) == cabi.TSKV_ERR_UNSUPPORTED
    assert sw.increase_status(truth, q, {}) == cabi.TSKV_ERR_UNSUPPORTED
    assert sw.increase_status({0: []}, q, {}) is None
    assert sw.increase_status(truth, QueryOption([inc(1, I64)], series_ids=[1]), {}) is None
    assert sw.increase_status(truth, QueryOption([inc(1, I64)], group_by_series=True), {}) is None
    # a group map decides alone: one selected series per group is accepted without GROUP BY series
    q1 = QueryOption([inc(1, I64)], series_ids=[0, 1])
    assert sw.increase_status(truth, q1, {"group_ids": np.array([0, 1], dtype=np.uint32)}) is None


@pytest.mark.parametrize("index", range(0, N_INC_CASES, 5))
def test_increase_validity_is_count(index):
    """Every increase of an accepted random increase case is valid exactly where COUNT(c) > 0 of the independent exact
    reference."""
    case = sw.random_increase_case(index, BASE_SEED)
    if sw.increase_status(case.truth, case.query, case.extra) is not None:
        return
    kw = dict(tombstones=case.tombstones, files=case.files, group_ids=case.extra.get("group_ids"),
              edges=case.extra.get("edges"))
    for col in sorted({c.column_id for c in case.query.columns if c.increase}):
        count = count_result(case, col)
        if count is None:
            return
        _, ok, _ = exact_increase_cells(case.truth, case.query, col, sw.COLUMNS[col], count.size, **kw)
        np.testing.assert_array_equal(ok, count > 0, err_msg="%s column %d" % (case.describe(), col))
