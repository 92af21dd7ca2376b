"""The exact reference for GROUP BY tags (tests/group_reference.py exact_aggregate_grouped) checked on its own (no
GPU): its COUNT / wrapping SUM / MIN / MAX equal the oracle's per-series results folded by group."""
import numpy as np
import pytest

from cnosdb_b200 import cabi
from oracle import pyoracle as orc
from tests.group_reference import exact_aggregate_grouped
from tests.helpers import (GEOM_AGGS, GEOM_FIELDS, GEOMETRY_CASES, ReferenceError, _okey, _okey_inv, exact_fit_grid,
                           geometry_arena, make_query, random_arena)

FIELDS = ((1, cabi.TSKV_PT_I64), (2, cabi.TSKV_PT_F64), (3, cabi.TSKV_PT_U64))


def fold_by_group(per_series, group_ids, n_groups):
    """{(column, agg): (values [n_groups, n_buckets], validity)} of COUNT / SUM / MIN / MAX from a group_by_series
    result, slot s folded into group group_ids[s] (integer sums wrap; f64 sums are left out)."""
    out = {}
    gid = np.asarray(group_ids, dtype=np.int64)
    for col, agg in per_series.names:
        if agg not in ("count", "sum", "min", "max"):
            continue
        pt = per_series.phys[col]
        if agg == "sum" and pt == cabi.TSKV_PT_F64:
            continue
        v, ok = per_series.column(col, agg)
        cnt = per_series.column(col, "count")[0].astype(np.uint64)
        gc = np.zeros((n_groups, cnt.shape[1]), dtype=np.uint64)
        np.add.at(gc, gid, cnt)
        have = gc > 0
        if agg == "count":
            out[(col, agg)] = (gc, np.ones_like(have))
        elif agg == "sum":
            s = np.zeros((n_groups, cnt.shape[1]), dtype=np.uint64)
            with np.errstate(over="ignore"):
                np.add.at(s, gid, np.where(ok, v, 0).view(np.uint64))
            out[(col, agg)] = (s, have)
        else:
            big = np.iinfo(np.int64).max if agg == "min" else np.iinfo(np.int64).min
            key = np.where(ok, _okey(pt, v.reshape(-1)).reshape(v.shape), big)
            k = np.full((n_groups, cnt.shape[1]), big, dtype=np.int64)
            (np.minimum if agg == "min" else np.maximum).at(k, gid, key)
            out[(col, agg)] = (np.where(have, _okey_inv(pt, k.reshape(-1)).reshape(k.shape), 0).astype(np.uint64), have)
    return out


def assert_exact_folds(exp, folded, what):
    for (col, agg), (v, ok) in folded.items():
        j = exp.names.index((col, agg))
        ev = exp.validity[j].reshape(v.shape)
        assert (ev == ok).all(), "%s: %s %s validity" % (what, col, agg)
        assert (exp.values[j].reshape(v.shape)[ok] == v[ok]).all(), "%s: %s %s" % (what, col, agg)


def _maps(rng, n_slots):
    yield "one group", np.zeros(n_slots, dtype=np.uint32), 1
    yield "identity", np.arange(n_slots, dtype=np.uint32), n_slots
    for g in (2, 7, max(1, n_slots // 3)):
        yield "random G=%d" % (g + 2), rng.integers(0, g, n_slots).astype(np.uint32), g + 2  # two groups stay empty


def test_grouped_reference_against_folded_oracle_random_arena():
    rng = np.random.default_rng(11)
    arena, descs, truth = random_arena(rng, n_series=30, n_points=300, fields=FIELDS, null_frac=0.15, jitter=400,
                                       multi_cg=True)
    sel = np.array(sorted(rng.choice(np.arange(30), 21, replace=False)), dtype=np.uint32)
    w = 40_000
    fbs, nb = exact_fit_grid(truth, w, 7, [(1_050_000, 1_200_000)])
    for ids in (None, sel):
        for preds in ([], [(1, cabi.TSKV_PT_I64, ">", -20)]):
            kw = dict(width=w, origin=7, first_bucket_start=fbs, n_buckets=nb, series_ids=ids, predicates=preds,
                      time_ranges=[(1_050_000, 1_200_000)])
            per_series = orc.scan_aggregate(arena, descs, make_query(FIELDS, GEOM_AGGS, group_by_series=True, **kw))
            n_slots = len(ids) if ids is not None else len(truth)
            for name, gmap, n_groups in _maps(rng, n_slots):
                exp = exact_aggregate_grouped(truth, make_query(FIELDS, GEOM_AGGS, **kw), gmap, n_groups)
                assert exp.n_groups == n_groups
                assert_exact_folds(exp, fold_by_group(per_series, gmap, n_groups), "%s sel=%s preds=%s" % (name, ids is not None, preds))


def test_grouped_reference_against_folded_oracle_geometry():
    rng = np.random.default_rng(12)
    for case in GEOMETRY_CASES[::9]:
        name, step, w, origin, t0, n, _ = case
        arena, descs, truth = geometry_arena(len(name), t0, step, n)
        fbs, nb = exact_fit_grid(truth, w, origin, [])
        if nb * len(truth) > 300_000:
            continue
        kw = dict(width=w, origin=origin, first_bucket_start=fbs, n_buckets=nb)
        try:
            per_series = orc.scan_aggregate(arena, descs, make_query(GEOM_FIELDS, GEOM_AGGS, group_by_series=True, **kw))
        except orc.OracleError as e:  # rows whose window start wraps: no bucket, with or without groups
            assert e.status == cabi.TSKV_ERR_BUCKET_RANGE
            with pytest.raises(ReferenceError):
                exact_aggregate_grouped(truth, make_query(GEOM_FIELDS, GEOM_AGGS, **kw), np.zeros(len(truth), dtype=np.uint32), 1)
            continue
        for gname, gmap, n_groups in _maps(rng, len(truth)):
            exp = exact_aggregate_grouped(truth, make_query(GEOM_FIELDS, GEOM_AGGS, **kw), gmap, n_groups)
            assert_exact_folds(exp, fold_by_group(per_series, gmap, n_groups), "%s %s" % (name, gname))
