"""f64 pages of IEEE special values and adversarial bit patterns through every Gorilla decoder of the scan (see
f64_edge_arena in tests/helpers.py): GorillaCursor (k_decode_warp), GorillaRing (every fused
bin, k_build_skip's restart points, pages cut into parts), next to the raw twin of every page. COUNT / MIN / MAX (IEEE totalOrder, so the NaN keys 0x7FFF...FFFF and 0xFFFF...FFFF are the MIN and MAX
identities) must equal the exact reference bit for bit, SUM / MEAN its class (NaN, the exact inf, or finite within the
order-free bound, +0.0 when zero), and FIRST / LAST the oracle bit for bit, NaN payloads included."""
import numpy as np
import pytest

from cnosdb_b200 import cabi, datagen
from oracle import pyoracle as orc
from tests.helpers import (ALL_AGGS, F64_FIELDS, F64_LENGTHS, F64_SERIES, F64_STEP, F64_T0, assert_matches_exact,
                           bucket_spec, exact_aggregate, f64_edge_arena, f64_edge_bits, f64_edge_expected,
                           f64_edge_queries, make_query)

pytestmark = pytest.mark.gpu

ENVS = ("1", "3")  # TSKV_PARTS


def _first_last_equal(got, exp, what):
    for j, (col, agg) in enumerate(got.names):
        if agg in ("first", "last"):
            assert (got.validity[j] == exp.validity[j]).all(), "%s col %s %s validity" % (what, col, agg)
            bad = np.nonzero(got.values[j] != exp.values[j])[0]
            assert bad.size == 0, "%s col %s %s at %s: got %s exp %s" % (
                what, col, agg, bad[:5], [hex(x) for x in got.values[j][bad[:3]]], [hex(x) for x in exp.values[j][bad[:3]]])


def _twins_equal(got, what):
    """Column 1 (Gorilla) and column 2 (raw) hold the same rows: COUNT / MIN / MAX / FIRST / LAST agree bit for bit."""
    for j, (col, agg) in enumerate(got.names):
        if col == 1 and agg in ("count", "min", "max", "first", "last"):
            k = got.names.index((2, agg))
            assert (got.values[j] == got.values[k]).all() and (got.validity[j] == got.validity[k]).all(), \
                "%s: %s of the Gorilla and the raw page differ" % (what, agg)


def _check(got, exp, ora, what):
    assert_matches_exact(got, exp, what=what)
    _twins_equal(got, what)
    if ora is not None:
        _first_last_equal(got, ora, what)


@pytest.mark.parametrize("n", F64_LENGTHS)
def test_f64_edges(engine, n, monkeypatch):
    arena, descs, truth = f64_edge_arena(n, n)
    pages = engine.upload_pages(arena, descs)
    # the pages decode to the generated bit patterns (GorillaCursor / the raw decoder)
    dec = engine.decode_pages(pages, descs)
    for k, d in enumerate(descs):
        if d["phys_type"] == cabi.TSKV_PT_F64:
            ts, cols = truth[int(d["series_id"])][0]
            vals, valid = cols[int(d["column_id"])]
            v, ok = dec[k]
            assert (ok == valid).all() and (v[valid] == vals.view(np.uint64)[valid]).all(), \
                "n=%d: page %d (series %d column %d) decodes to other bits" % (n, k, d["series_id"], d["column_id"])
    hp = engine.upload_pages(arena, descs, host_resident=True)  # no restart points, pages pulled over PCIe
    for name, q, extra in f64_edge_queries(n):
        exp = f64_edge_expected(truth, q, extra)
        sel = any(c.agg_mask & (cabi.TSKV_AGG_FIRST | cabi.TSKV_AGG_LAST) for c in q.columns)
        ora = orc.scan_aggregate(arena, descs, q) if sel else None
        kw = dict(slide=extra.get("slide"), group_ids=extra.get("group_ids"), n_groups=extra.get("n_groups"))
        for parts in ENVS:
            monkeypatch.setenv("TSKV_PARTS", parts)
            what = "n=%d %s parts=%s" % (n, name, parts)
            _check(engine.scan_aggregate(pages, q, **kw), exp, ora, what)
        monkeypatch.setenv("TSKV_PARTS", ENVS[0])
        _check(engine.scan_aggregate(hp, q, **kw), exp, ora, "n=%d %s host-resident" % (n, name))
        if name == "bucket+sel":  # a second pass of a prepared scan replays its graph
            s = engine.prepare(pages, q)
            s.run()
            s.enqueue()
            s.sync()
            _check(s.finalize(), exp, ora, "n=%d %s replay" % (n, name))
            s.close()
    hp.close()
    pages.close()


def test_f64_edges_through_the_overlap_merge(engine):
    """Two chunk files of each series whose rows interleave (k_merge_chunks): the merged rows' sums, keys and FIRST /
    LAST."""
    rng = np.random.default_rng(17)
    b = datagen.ArenaBuilder()
    truth, files = {}, []
    ids = range(0, 20)  # one series of every value kind, with and without nulls
    for sid in ids:
        for f in range(2):
            m = 300
            ts = F64_T0 + (2 * np.arange(m, dtype=np.int64) + f) * F64_STEP  # file 0 even rows, file 1 odd rows
            vals = f64_edge_bits(rng, sid, m).view(np.float64)
            valid = rng.random(m) >= 0.25 if sid % 7 == 3 else np.ones(m, dtype=bool)
            vv = None if valid.all() else valid
            b.add_column_group(sid, ts, [(1, cabi.TSKV_PT_F64, vals, vv), (2, cabi.TSKV_PT_F64, vals, vv, datagen.encode_raw)])
            truth.setdefault(sid, []).append((ts, {1: (vals, valid), 2: (vals, valid)}))
            files.append(f + 1)
    arena, descs = b.finish()
    pages = engine.upload_pages(arena, descs)
    pages.set_chunk_files(files)
    w = 50 * F64_STEP
    fbs, nb = bucket_spec(F64_T0, F64_T0 + 600 * F64_STEP, w)
    for gbs in (True, False):
        sids = None if gbs else np.array([s for s in ids if s % 10 not in (8,)], dtype=np.uint32)
        q = make_query(F64_FIELDS, ALL_AGGS, width=w, first_bucket_start=fbs, n_buckets=nb, group_by_series=gbs,
                       series_ids=sids)
        exp = exact_aggregate(truth, q, files=files)
        ora = orc.scan_aggregate(arena, descs, q, chunk_files=files)
        _check(engine.scan_aggregate(pages, q), exp, ora, "overlap merge gbs=%s" % gbs)
    pages.close()


def test_f64_edges_through_a_two_shard_exchange(engine):
    """Two series shards scanned separately and merged like an all-gather on one device (k_merge_gathered): NaN, inf
    and the totalOrder keys across ranks."""
    import torch
    from cnosdb_b200.parallel import device_tensor
    n = 257
    _, _, truth = f64_edge_arena(n, n)
    name, q, _ = f64_edge_queries(n)[0]  # GROUP BY bucket, every series but the DBL_MAX ones
    ids = [int(s) for s in q.series_ids]
    exp = exact_aggregate(truth, q)
    dev = torch.device("cuda", engine.device)
    scans, regions, keep = [], [], []
    for part in (ids[::2], ids[1::2]):  # interleaved: both shards hold every value kind
        b = datagen.ArenaBuilder()
        for s in part:
            ts, cols = truth[s][0]
            vals, valid = cols[1]
            vv = None if valid.all() else valid
            b.add_column_group(s, ts, [(1, cabi.TSKV_PT_F64, vals, vv), (2, cabi.TSKV_PT_F64, vals, vv, datagen.encode_raw)])
        arena, descs = b.finish()
        pages = engine.upload_pages(arena, descs)
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
        assert_matches_exact(got, exp, what="2-shard exchange")
        _twins_equal(got, "2-shard exchange")
        s.close()
    for pages in keep:
        pages.close()
