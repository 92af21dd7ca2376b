"""The fused scan's bucket arithmetic at the edges of its time geometry (see GEOMETRY_CASES in tests/helpers.py): steps
from 0 to 2^40 + 3, widths that are and are not multiples of the step, narrower than it, up to 2^63 - 1, origins that are
negative or >= the width, rows on both sides of the truncating-% regime and at the i64 limits, and time ranges on, beside
and between rows and bucket edges. Every query runs with pages whole and cut into 3 parts, and every single-range query
runs again with its range split in two (two ranges turn the row-space fast path off): COUNT / SUM / MIN / MAX must be
bit-identical across the two and equal the exact reference. FIRST / LAST must equal the exact reference (which keeps the
known deviation at the i64 limits) and the oracle wherever a page's timestamps are distinct."""
import numpy as np
import pytest

from cnosdb_b200 import cabi
from cnosdb_b200.engine import TskvError
from oracle import pyoracle as orc
from tests.helpers import (GEOM_BLOCK, GEOMETRY_CASES, I64_MIN, ReferenceError, assert_matches_exact, exact_aggregate,
                           geometry_arena, geometry_queries, geometry_ranges, sel_unsupported, split_ranges,
                           time_page_is_rle)

pytestmark = pytest.mark.gpu

ENVS = ("1", "3")  # TSKV_PARTS


def _scan(engine, pages, q):
    try:
        return engine.scan_aggregate(pages, q), None
    except TskvError as e:
        return None, e.status


def _first_last_equal(got, exp, what):
    for j, (col, agg) in enumerate(got.names):
        if agg in ("first", "last"):
            assert (got.validity[j] == exp.validity[j]).all(), "%s col %s %s validity" % (what, col, agg)
            bad = np.nonzero(got.values[j] != exp.values[j])[0]
            assert bad.size == 0, "%s col %s %s differs at %s" % (what, col, agg, bad[:5])


def _plain_equal(a, b, what):
    """COUNT / integer SUM / MIN / MAX of two GPU runs, bit for bit (an f64 sum depends on the order)."""
    for j, (col, agg) in enumerate(a.names):
        if agg in ("count", "min", "max") or (agg == "sum" and a.phys[col] != cabi.TSKV_PT_F64):
            assert (a.validity[j] == b.validity[j]).all() and (a.values[j] == b.values[j]).all(), \
                "%s col %s %s differs between one range and the split range" % (what, col, agg)


@pytest.mark.parametrize("case", GEOMETRY_CASES, ids=[c[0] for c in GEOMETRY_CASES])
def test_bucket_geometry(engine, case, monkeypatch):
    name, step, w, origin, t0, n, kinds = case
    arena, descs, truth = geometry_arena(len(name), t0, step, n)
    time_idx = np.nonzero(descs["phys_type"] == cabi.TSKV_PT_TIME)[0]
    # blocks A and B must really be run-length time pages (the writer picks the encoding)
    for k in time_idx:
        if descs[k]["series_id"] < 2 * GEOM_BLOCK and descs[k]["num_values"] >= 2:
            assert time_page_is_rle(arena, descs[k]), "series %d: time page is not RLE" % descs[k]["series_id"]
    pages = engine.upload_pages(arena, descs)
    # the time pages decode to the generated timestamps (k_decode_warp's RLE closed form at the same extremes)
    for k in time_idx:
        (v, ok), = engine.decode_pages(pages, descs, int(k), 1)
        sid = int(descs[k]["series_id"])
        assert ok.all() and (v.view(np.int64) == truth[sid][0][0]).all(), "%s: time page of series %d" % (name, sid)

    for kind in kinds:
        ranges = geometry_ranges(kind, t0, step, n, w, origin)
        for qname, q in geometry_queries(case, ranges, truth):
            variants = [ranges] + ([split_ranges(ranges)] if len(ranges) == 1 else [])
            sel = qname in ("bucket+sel", "by_series", "unbucketed")
            unsupported = sel_unsupported(q, truth)
            first = None
            for rs in variants:
                q.time_ranges = rs
                what = "%s %s %s ranges=%s" % (name, kind, qname, rs)
                try:
                    exp, err = exact_aggregate(truth, q), None
                except ReferenceError as e:
                    exp, err = None, e.status
                # FIRST / LAST against the oracle where a page's timestamps are distinct (the storage engine never
                # writes two rows of one series at the same time; with step 0 every row ties)
                # (with group_by_series the keys are raw row times, and a LAST at INT64_MIN equals the empty key: a known
                # deviation, DESIGN section 7)
                ora = orc.scan_aggregate(arena, descs, q) if (sel and step and err is None and not unsupported and
                                                               not (qname == "by_series" and t0 == I64_MIN)) else None
                for parts in ENVS:
                    monkeypatch.setenv("TSKV_PARTS", parts)
                    wh = "%s parts=%s" % (what, parts)
                    got, st = _scan(engine, pages, q)
                    if unsupported:
                        assert st == cabi.TSKV_ERR_UNSUPPORTED, wh
                        continue
                    if err is not None:
                        assert st == err, "%s: status %s, expected %s" % (wh, st, err)
                        continue
                    assert st is None, "%s: status %s" % (wh, st)
                    assert_matches_exact(got, exp, what=wh, first_last=bool(step))
                    if ora is not None:
                        _first_last_equal(got, ora, wh)
                    if first is None:
                        first = got
                    else:
                        _plain_equal(got, first, wh)

        if kind == "none":  # the exact grid one bucket short at either end: rows without a bucket
            q = geometry_queries(case, [], truth)[0][1]
            if q.n_buckets >= 2:
                for fbs in (q.first_bucket_start + w, q.first_bucket_start):
                    q.first_bucket_start, q.n_buckets = fbs, geometry_queries(case, [], truth)[0][1].n_buckets - 1
                    with pytest.raises(orc.OracleError) as oe:
                        orc.scan_aggregate(arena, descs, q)
                    assert oe.value.status == cabi.TSKV_ERR_BUCKET_RANGE
                    for parts in ENVS:
                        monkeypatch.setenv("TSKV_PARTS", parts)
                        assert _scan(engine, pages, q)[1] == cabi.TSKV_ERR_BUCKET_RANGE, "%s short grid %d" % (name, fbs)
    pages.close()
