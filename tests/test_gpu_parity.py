"""Parity of the CUDA path (through the C ABI) against the CPU oracle. Bit-exact for decode, counts,
integer aggregates and f64 min/max/first/last; f64 sum/mean within 1e-6 relative (BASELINE.md section 4)."""
import numpy as np
import pytest

from cnosdb_b200 import cabi, datagen
from cnosdb_b200.engine import PushedAggregate, QueryOption, TskvError
from oracle import pyoracle as orc
from tests.helpers import ALL_AGGS, assert_results_equal, bucket_spec, make_query, random_arena, time_page_is_rle

pytestmark = pytest.mark.gpu


def bits_to_f64(bits):
    return np.array([int(b, 16) for b in bits], dtype=np.uint64).view(np.float64)


def check_decode(engine, arena, descs):
    pages = engine.upload_pages(arena, descs)
    got = engine.decode_pages(pages, descs)
    exp = orc.decode_pages(arena, descs)
    assert len(got) == len(exp)
    for i, ((gv, gb), (ev, eb)) in enumerate(zip(got, exp)):
        assert (gb == eb).all(), "validity differs on page %d" % i
        assert (gv == ev).all(), "values differ on page %d: %s" % (i, np.nonzero(gv != ev)[0][:5])
    pages.close()


def test_decode_golden_corpora(engine, golden):
    """Every reference codec corpus, decoded on the GPU, bit-exact (incl. NaN payloads)."""
    g = golden["codec_vectors"]
    b = datagen.ArenaBuilder()
    sid = 0

    def add(pt, data, n):
        nonlocal sid
        b.add_page(datagen.build_page(datagen.encode_timestamps(np.arange(n)), n), sid, 0, cabi.TSKV_PT_TIME, n)
        b.add_page(datagen.build_page(data, n), sid, 1, pt, n)
        sid += 1

    for grp in ("i64_rle", "i64_simple8b"):
        for t in g[grp]["tests"]:
            add(cabi.TSKV_PT_I64, datagen.encode_integers(t["input"]), len(t["input"]))
    add(cabi.TSKV_PT_I64, datagen.encode_integers(g["i64_uncompressed"]["input"]), 4)
    add(cabi.TSKV_PT_I64, datagen.encode_integers(np.full(509, 809201799168)), 509)
    add(cabi.TSKV_PT_I64, datagen.encode_integers([346]), 1)
    for grp in ("ts_rle", "ts_simple8b"):
        for t in g[grp]["tests"]:  # timestamp codec on an i64 column (Encoding::DeltaTs, instance.rs:379)
            add(cabi.TSKV_PT_I64, datagen.encode_timestamps(t["input"]), len(t["input"]))
            add(cabi.TSKV_PT_TIME, datagen.encode_timestamps(t["input"]), len(t["input"]))
    add(cabi.TSKV_PT_TIME, datagen.encode_timestamps(g["ts_uncompressed"]["input"]), 4)
    add(cabi.TSKV_PT_TIME, datagen.encode_integers(g["ts_uncompressed"]["input"]), 4)  # Delta on a time column
    for t in g["u64_rle"]["tests"] + g["u64_simple8b"]["tests"]:
        add(cabi.TSKV_PT_U64, datagen.encode_integers(np.array(t["input"], dtype=np.uint64).view(np.int64)), len(t["input"]))
    add(cabi.TSKV_PT_U64, datagen.encode_integers(np.full(1000, 1232342341234)), 1000)
    for t in g["f64_roundtrip"]["tests"]:
        v = bits_to_f64(t["input_bits"])
        add(cabi.TSKV_PT_F64, datagen.encode_floats(v), len(v))
    v = bits_to_f64(g["f64_special_values"]["input_bits"])
    add(cabi.TSKV_PT_F64, datagen.encode_floats(v), len(v))
    add(cabi.TSKV_PT_F64, datagen.encode_raw(v.view(np.uint64)), len(v))  # Encoding::Null
    add(cabi.TSKV_PT_I64, datagen.encode_raw(np.arange(7, dtype=np.uint64)), 7)
    arena, descs = b.finish()
    check_decode(engine, arena, descs)


def test_decode_simple8b_all_widths_and_runs(engine):
    rng = np.random.default_rng(231)
    b = datagen.ArenaBuilder()
    cases = []
    for bits in (1, 2, 3, 4, 5, 6, 7, 8, 10, 12, 15, 20, 30, 59):
        cases.append(np.cumsum(rng.integers(0, 2**bits, 1000).astype(np.int64) // 2 * rng.choice([-1, 1], 1000)))
    cases.append(np.cumsum(np.ones(1000, dtype=np.int64)) * -1)   # zigzag(−1) = 1: runs of ones → selectors 0/1
    ones = np.ones(500, dtype=np.int64) * -1
    ones[119] = 5
    ones[240] = 9
    cases.append(np.cumsum(ones))
    cases.append(rng.integers(-2**62, 2**62, 300))                # raw
    for i, v in enumerate(cases):
        b.add_column_group(i, np.arange(len(v)), [(1, cabi.TSKV_PT_I64, v, None)])
    arena, descs = b.finish()
    check_decode(engine, arena, descs)


def test_decode_c1_shape(engine):
    """BASELINE config C1: 1 series x 10 000 i64, Delta (zigzag + simple8b) decode only, seed 1."""
    g = datagen.generate(1, n_fields=1, n_points=10_000, value_kind=datagen.I64_WALK, seed=1)
    check_decode(engine, g.arena, g.descs)
    # forced RLE (constant step) and raw (|delta| >= 2^59) sub-cases
    b = datagen.ArenaBuilder()
    b.add_column_group(0, np.arange(10_000) * 10, [(1, cabi.TSKV_PT_I64, np.arange(10_000) * 3 - 7, None)])
    big = (np.arange(10_000, dtype=np.int64) % 2) * (2**61) - 2**60
    b.add_column_group(1, np.arange(10_000) * 10, [(1, cabi.TSKV_PT_I64, big, None)])
    arena, descs = b.finish()
    check_decode(engine, arena, descs)


def test_decode_nulls_and_generated_mix(engine):
    g = datagen.generate(200, n_fields=3, n_points=1000, value_kind=datagen.MIXED, seed=4, jitter_permille=300,
                         jitter_max=999_999, null_page_permille=300, null_row_permille=50, raw_encoding_permille=100)
    check_decode(engine, g.arena, g.descs)
    rng = np.random.default_rng(7)
    arena, descs, _ = random_arena(rng, n_series=30, n_points=257, null_frac=0.4,
                                   fields=((1, cabi.TSKV_PT_I64), (2, cabi.TSKV_PT_F64), (3, cabi.TSKV_PT_U64)))
    check_decode(engine, arena, descs)


def test_decode_empty_and_all_null_pages(engine):
    b = datagen.ArenaBuilder()
    b.add_column_group(0, np.arange(40), [(1, cabi.TSKV_PT_I64, np.arange(40), np.zeros(40, dtype=bool)),
                                          (2, cabi.TSKV_PT_F64, np.arange(40.0), np.zeros(40, dtype=bool))])
    v = np.zeros(9, dtype=bool)
    v[4] = True
    b.add_column_group(1, np.arange(9), [(1, cabi.TSKV_PT_I64, np.arange(9), v), (2, cabi.TSKV_PT_F64, np.arange(9.0), v)])
    arena, descs = b.finish()
    check_decode(engine, arena, descs)


SCAN_FIELDS = ((1, cabi.TSKV_PT_I64), (2, cabi.TSKV_PT_F64), (3, cabi.TSKV_PT_U64))


@pytest.mark.parametrize("group_by_series", [False, True])
@pytest.mark.parametrize("variant", ["plain", "nulls", "jitter", "multi_cg", "raw"])
def test_scan_parity_small(engine, group_by_series, variant):
    rng = np.random.default_rng(hash((variant, group_by_series)) % 2**32)
    kw = dict(n_series=70, n_points=333, fields=SCAN_FIELDS)
    if variant == "nulls":
        kw["null_frac"] = 0.2
    if variant == "jitter":
        kw["jitter"] = 300
    if variant == "multi_cg":
        kw.update(multi_cg=True, null_frac=0.05)
    if variant == "raw":
        kw["raw_frac"] = 0.5
    arena, descs, _ = random_arena(rng, **kw)
    pages = engine.upload_pages(arena, descs)
    sel = np.array(sorted(rng.choice(np.arange(80), 45, replace=False)), dtype=np.uint32)
    t_lo, t_hi = 1_000_000 + 20_500, 1_000_000 + 300_000
    fbs, nb = bucket_spec(t_lo, t_hi, 17_000, origin=3)
    for series_ids in (sel, None):
        for ranges in ([(t_lo, t_hi)], [(t_lo, t_lo + 50_000), (t_lo + 90_000, t_hi)], []):
            if not ranges:
                lo = 1_000_000 - 400
                hi = int(max(int(descs["num_values"].max()) * 2 * 1000 + 1_000_000 + 400, t_hi))
                f2, n2 = bucket_spec(lo, hi, 17_000, origin=3)
                q = make_query(SCAN_FIELDS, series_ids=series_ids, time_ranges=[], origin=3, width=17_000,
                               first_bucket_start=f2, n_buckets=n2, group_by_series=group_by_series)
            else:
                q = make_query(SCAN_FIELDS, series_ids=series_ids, time_ranges=ranges, origin=3, width=17_000,
                               first_bucket_start=fbs, n_buckets=nb, group_by_series=group_by_series)
            got = engine.scan_aggregate(pages, q)
            exp, pts = orc.scan_aggregate(arena, descs, q, return_points=True)
            assert_results_equal(got, exp, what="%s %s" % (variant, ranges))
            assert engine.counters()["points_decoded"] == pts
    # unbucketed: one cell per group
    q = make_query(SCAN_FIELDS, series_ids=sel, time_ranges=[(t_lo, t_hi)], group_by_series=group_by_series)
    assert_results_equal(engine.scan_aggregate(pages, q), orc.scan_aggregate(arena, descs, q), what="unbucketed")
    pages.close()


def test_scan_c2_shape(engine):
    """BASELINE C2 (scaled to 2 000 series for the oracle): f64 Gorilla, closed range rows 250..749, sum+count."""
    for kind in (datagen.F64_INT, datagen.F64_NOISE):
        g = datagen.generate(2000, n_fields=1, n_points=1000, value_kind=kind, seed=2)
        pages = engine.upload_pages(g.arena, g.descs)
        lo, hi = datagen.TSBS_T0 + 250 * datagen.TSBS_STEP, datagen.TSBS_T0 + 749 * datagen.TSBS_STEP
        for gbs in (True, False):
            q = QueryOption([PushedAggregate(1, cabi.TSKV_PT_F64, ["sum", "count"])], time_ranges=[(lo, hi)],
                            group_by_series=gbs)
            got, exp = engine.scan_aggregate(pages, q), orc.scan_aggregate(g.arena, g.descs, q, n_threads=8)
            assert_results_equal(got, exp, what="C2")
            assert (got.column(1, "count")[0] == (500 if gbs else 500 * 2000)).all()
        pages.close()


def test_scan_c3_shape(engine):
    """BASELINE C3 (scaled to 3 000 hosts): 10 fields, 1-min mean/max over 167 buckets."""
    for kind, pt in ((datagen.I64_WALK, cabi.TSKV_PT_I64), (datagen.F64_INT, cabi.TSKV_PT_F64)):
        g = datagen.generate(3000, n_fields=10, n_points=1000, value_kind=kind, seed=3)
        pages = engine.upload_pages(g.arena, g.descs)
        w = 60_000_000_000
        fbs, nb = bucket_spec(datagen.TSBS_T0, datagen.TSBS_T0 + 999 * datagen.TSBS_STEP, w)
        assert nb == 167
        q = QueryOption([PushedAggregate(c, pt, ["mean", "max"]) for c in range(1, 11)], width=w,
                        first_bucket_start=fbs, n_buckets=nb)
        got, exp = engine.scan_aggregate(pages, q), orc.scan_aggregate(g.arena, g.descs, q, n_threads=8)
        assert_results_equal(got, exp, what="C3")
        assert engine.counters()["points_decoded"] == 3000 * 10 * 1000
        pages.close()


def test_scan_c4_shape(engine):
    """BASELINE C4 (scaled to 20 000 series): mixed i64/f64, 20% jittered timestamps, 1% pages with 5% nulls,
    10% tag selection (hash(id) % 10 == 0), group by 1-min bucket."""
    g = datagen.generate(20_000, n_fields=1, n_points=1000, value_kind=datagen.MIXED, seed=4, jitter_permille=200,
                         jitter_max=999_999, null_page_permille=10, null_row_permille=50)
    pages = engine.upload_pages(g.arena, g.descs)
    ids = np.arange(20_000, dtype=np.uint64)
    sel = ids[((ids * np.uint64(0x9E3779B97F4A7C15)) >> np.uint64(32)) % np.uint64(10) == 0].astype(np.uint32)
    w = 60_000_000_000
    fbs, nb = bucket_spec(datagen.TSBS_T0 - 1_000_000, datagen.TSBS_T0 + 999 * datagen.TSBS_STEP + 1_000_000, w)
    # even ids carry the i64 column 1, odd ids the f64 column 2 (a column absent from a group is skipped)
    q = QueryOption([PushedAggregate(1, cabi.TSKV_PT_I64, ALL_AGGS), PushedAggregate(2, cabi.TSKV_PT_F64, ALL_AGGS)],
                    series_ids=sel, width=w, first_bucket_start=fbs, n_buckets=nb)
    got, exp = engine.scan_aggregate(pages, q), orc.scan_aggregate(g.arena, g.descs, q, n_threads=8)
    assert_results_equal(got, exp, what="C4")
    assert engine.counters()["points_decoded"] > 0.99 * len(sel) * 1000
    # the same scan with the pages left in host memory (PCIe gather of the selected pages per query)
    hp = engine.upload_pages(g.arena, g.descs, host_resident=True)
    assert_results_equal(engine.scan_aggregate(hp, q), exp, what="C4 host-resident")
    assert engine.counters()["page_read_bytes"] < 0.2 * g.arena.size
    hp.close()
    pages.close()


def test_scan_c5_shape(engine):
    """BASELINE C5 (scaled): last point per series + 5-min window max over the last hour (360 pts, 12 buckets)."""
    g = datagen.generate(5000, n_fields=5, n_points=360, value_kind=datagen.I64_WALK, seed=5)
    pages = engine.upload_pages(g.arena, g.descs)
    cols = [PushedAggregate(c, cabi.TSKV_PT_I64, ["last"]) for c in range(1, 6)]
    q = QueryOption(cols, group_by_series=True)
    assert_results_equal(engine.scan_aggregate(pages, q), orc.scan_aggregate(g.arena, g.descs, q, n_threads=8), what="C5 last")
    w = 300_000_000_000
    fbs, nb = bucket_spec(datagen.TSBS_T0, datagen.TSBS_T0 + 359 * datagen.TSBS_STEP, w)
    assert nb == 12
    q = QueryOption([PushedAggregate(c, cabi.TSKV_PT_I64, ["max"]) for c in range(1, 6)], width=w,
                    first_bucket_start=fbs, n_buckets=nb)
    assert_results_equal(engine.scan_aggregate(pages, q), orc.scan_aggregate(g.arena, g.descs, q, n_threads=8), what="C5 max")
    pages.close()


def test_full_size_properties(engine):
    """Size-independent properties at a larger size than the oracle is run on: counts sum to the number of
    in-range rows, sum over buckets == unbucketed sum (i64, exact), per-series totals == global totals."""
    n_series = 50_000
    g = datagen.generate(n_series, n_fields=2, n_points=1000, value_kind=datagen.I64_WALK, seed=11)
    pages = engine.upload_pages(g.arena, g.descs)
    w = 60_000_000_000
    fbs, nb = bucket_spec(datagen.TSBS_T0, datagen.TSBS_T0 + 999 * datagen.TSBS_STEP, w)
    cols = [PushedAggregate(c, cabi.TSKV_PT_I64, ["count", "sum", "min", "max"]) for c in (1, 2)]
    rb = engine.scan_aggregate(pages, QueryOption(cols, width=w, first_bucket_start=fbs, n_buckets=nb))
    assert engine.counters()["points_decoded"] == n_series * 2 * 1000
    ru = engine.scan_aggregate(pages, QueryOption(cols))
    rs = engine.scan_aggregate(pages, QueryOption(cols, group_by_series=True))
    for c in (1, 2):
        assert rb.column(c, "count")[0].sum() == n_series * 1000 == ru.column(c, "count")[0][0, 0]
        assert rb.column(c, "sum")[0].sum() == ru.column(c, "sum")[0][0, 0] == rs.column(c, "sum")[0].sum()
        assert rb.column(c, "min")[0].min() == ru.column(c, "min")[0][0, 0] == rs.column(c, "min")[0].min()
        assert rb.column(c, "max")[0].max() == ru.column(c, "max")[0][0, 0] == rs.column(c, "max")[0].max()
        assert (rs.column(c, "count")[0] == 1000).all()
    pages.close()


def test_first_last_semantics_match_reference_rules(engine):
    b = datagen.ArenaBuilder()
    ts = np.array([10, 20, 30, 40], dtype=np.int64)
    b.add_column_group(1, ts, [(1, cabi.TSKV_PT_I64, np.array([1, 2, 3, 4]), np.array([False, True, True, True]))])
    b.add_column_group(2, ts + 1, [(1, cabi.TSKV_PT_I64, np.array([5, 6, 7, 8]), None)])
    for sid, (a, z) in enumerate([(11, 12), (21, 22), (31, 32)]):
        b.add_column_group(sid + 5, np.array([100, 200]), [(2, cabi.TSKV_PT_F64, np.array([a, z], dtype=np.float64), None)])
    arena, descs = b.finish()
    pages = engine.upload_pages(arena, descs)
    q = QueryOption([PushedAggregate(1, cabi.TSKV_PT_I64, ["first", "last", "count"]),
                     PushedAggregate(2, cabi.TSKV_PT_F64, ["first", "last"])])
    got = engine.scan_aggregate(pages, q)
    assert_results_equal(got, orc.scan_aggregate(arena, descs, q))
    assert got.column(1, "first")[0][0, 0] == 5 and got.column(2, "first")[0][0, 0] == 11.0
    assert got.column(2, "last")[0][0, 0] == 12.0
    pages.close()


def test_negative_timestamps_keep_the_window_quirk(engine):
    rng = np.random.default_rng(17)
    b = datagen.ArenaBuilder()
    for sid in range(20):
        ts = np.sort(rng.choice(np.arange(-4000, 3000), 150, replace=False)).astype(np.int64)
        b.add_column_group(sid, ts, [(1, cabi.TSKV_PT_I64, rng.integers(-9, 10, 150), None)])
    arena, descs = b.finish()
    pages = engine.upload_pages(arena, descs)
    w, origin = 500, 130
    fbs, _ = orc.sliding_window(-4000, w, w, origin)
    last, _ = orc.sliding_window(3000, w, w, origin)
    nb = (last - fbs) // w + 1
    q = make_query([(1, cabi.TSKV_PT_I64)], origin=origin, width=w, first_bucket_start=fbs, n_buckets=nb)
    assert_results_equal(engine.scan_aggregate(pages, q), orc.scan_aggregate(arena, descs, q), what="negative ts")
    pages.close()


def _corrupt(arena, descs, page_idx, fn):
    a = arena.copy()
    d = descs[page_idx]
    off, size, n = int(d["offset"]), int(d["size"]), int(d["num_values"])
    data_off = off + 16 + (n + 7) // 8
    fn(a, off, data_off, size)
    # re-seal the CRC so that the decoder (not the checksum) sees the corruption
    crc = orc.crc32(a[data_off:off + size])
    a[off + 12:off + 16] = np.frombuffer(int(crc).to_bytes(4, "big"), dtype=np.uint8)
    return a


@pytest.mark.parametrize("case,status", [
    ("bad_sub_encoding", cabi.TSKV_ERR_BAD_ENCODING),
    ("quantile", cabi.TSKV_ERR_UNSUPPORTED),
    ("truncated_gorilla", cabi.TSKV_ERR_SHORT_BLOCK),
    ("too_few_values", cabi.TSKV_ERR_BITSET_MISMATCH),
])
def test_decode_errors_match_oracle(engine, case, status):
    b = datagen.ArenaBuilder()
    n = 64
    b.add_column_group(0, np.arange(n), [(1, cabi.TSKV_PT_I64, np.cumsum(np.arange(n) % 7), None),
                                         (2, cabi.TSKV_PT_F64, np.arange(n) * 1.25 + 0.1, None)])
    arena, descs = b.finish()
    if case == "bad_sub_encoding":
        a = _corrupt(arena, descs, 1, lambda a, off, d, size: a.__setitem__(d + 1, 0x30))
        bad = 1
    elif case == "quantile":
        a = _corrupt(arena, descs, 1, lambda a, off, d, size: a.__setitem__(d, 3))
        bad = 1
    elif case == "truncated_gorilla":
        # keep the framing but zero the tail of the stream: the sentinel disappears
        a = _corrupt(arena, descs, 2, lambda a, off, d, size: a.__setitem__(slice(off + size - 40, off + size), 0))
        bad = 2
    else:
        # claim more valid rows than there are encoded values: shrink data by one simple8b word
        bb = datagen.ArenaBuilder()
        v = np.cumsum(np.arange(n) % 7)
        data = datagen.encode_integers(v)[:-8]
        bb.add_page(datagen.build_page(datagen.encode_timestamps(np.arange(n)), n), 0, 0, cabi.TSKV_PT_TIME, n)
        bb.add_page(datagen.build_page(data, n), 0, 1, cabi.TSKV_PT_I64, n)
        a, descs = bb.finish()
        bad = 1
    with pytest.raises(orc.OracleError) as oe:
        orc.decode_pages(a, descs)
    assert oe.value.status == status
    pages = engine.upload_pages(a, descs)
    with pytest.raises(TskvError) as ge:
        engine.decode_pages(pages, descs)
    assert ge.value.status == status and ge.value.page == bad
    pt = int(descs[bad]["phys_type"])
    with pytest.raises(TskvError) as se:
        engine.scan_aggregate(pages, QueryOption([PushedAggregate(int(descs[bad]["column_id"]), pt, ["count"])]))
    assert se.value.status == status
    pages.close()


def test_crc_mismatch_is_detected_at_upload(engine):
    g = datagen.generate(10, n_fields=1, n_points=100, seed=8)
    a = g.arena.copy()
    a[int(g.descs[3]["offset"]) + int(g.descs[3]["size"]) - 1] ^= 0x40
    with pytest.raises(TskvError) as e:
        engine.upload_pages(a, g.descs)
    assert e.value.status == cabi.TSKV_ERR_CRC_MISMATCH and e.value.page == 3
    engine.upload_pages(a, g.descs, verify_crc=False).close()


def test_query_validation_errors(engine):
    g = datagen.generate(10, n_fields=1, n_points=100, seed=8)
    pages = engine.upload_pages(g.arena, g.descs)
    with pytest.raises(TskvError) as e:   # rows outside the bucket range
        engine.scan_aggregate(pages, make_query([(1, cabi.TSKV_PT_I64)], width=1000, first_bucket_start=datagen.TSBS_T0, n_buckets=2))
    assert e.value.status == cabi.TSKV_ERR_BUCKET_RANGE
    with pytest.raises(TskvError) as e:   # wrong column type
        engine.scan_aggregate(pages, make_query([(1, cabi.TSKV_PT_F64)]))
    assert e.value.status == cabi.TSKV_ERR_INVALID_ARG
    with pytest.raises(TskvError) as e:   # unsorted selection
        engine.scan_aggregate(pages, make_query([(1, cabi.TSKV_PT_I64)], series_ids=np.array([3, 1], dtype=np.uint32)))
    assert e.value.status == cabi.TSKV_ERR_INVALID_ARG
    # a selection that matches nothing gives empty (invalid) cells and count 0
    r = engine.scan_aggregate(pages, make_query([(1, cabi.TSKV_PT_I64)], series_ids=np.array([77], dtype=np.uint32)))
    assert r.column(1, "count")[0][0, 0] == 0 and not r.column(1, "sum")[1][0, 0]
    pages.close()


def test_two_shard_exchange_matches_whole_scan(engine):
    """The multi-GPU exchange on one device: two contiguous series shards scanned separately with the
    GLOBAL selection list, their exchange regions concatenated like an all-gather, merged with
    tskvgpu_scan_merge_gathered -> identical to the oracle on the whole arena (incl. first/last ties)."""
    import torch
    from cnosdb_b200.parallel import device_tensor, select_tag_subset, shard_range
    n = 3000
    full = datagen.generate(n, n_fields=1, n_points=400, value_kind=datagen.MIXED, seed=31, jitter_permille=300,
                            jitter_max=999, null_page_permille=100, null_row_permille=200)
    sel = select_tag_subset(n, 3)
    w = 60_000_000_000
    fbs, nb = bucket_spec(datagen.TSBS_T0 - 1000, datagen.TSBS_T0 + 399 * datagen.TSBS_STEP + 1000, w)
    q = QueryOption([PushedAggregate(1, cabi.TSKV_PT_I64, ALL_AGGS), PushedAggregate(2, cabi.TSKV_PT_F64, ALL_AGGS)],
                    series_ids=sel, width=w, first_bucket_start=fbs, n_buckets=nb)
    exp = orc.scan_aggregate(full.arena, full.descs, q)
    dev = torch.device("cuda", engine.device)
    scans, regions, keep = [], [], []
    for r in range(2):
        lo, hi = shard_range(n, r, 2)
        g = datagen.generate(hi - lo, n_fields=1, n_points=400, value_kind=datagen.MIXED, seed=31, first_series_id=lo,
                             jitter_permille=300, jitter_max=999, null_page_permille=100, null_row_permille=200)
        pages = engine.upload_pages(g.arena, g.descs)
        s = engine.prepare(pages, q)
        s.run()
        ptr, words = s.exchange_view()
        regions.append(device_tensor(ptr, words, torch.int64, dev).clone())
        scans.append(s)
        keep.append((g, pages))
    gathered = torch.cat(regions)
    torch.cuda.synchronize()
    for s in scans:  # every rank merges the same gathered buffer
        s.merge_gathered(gathered.data_ptr(), 2)
        assert_results_equal(s.finalize(), exp, what="2-shard exchange")
        s.close()
    for _, pages in keep:
        pages.close()


@pytest.mark.parametrize("gbs", [False, True])
def test_short_jittered_pages_with_nulls_agree_with_oracle(engine, gbs):
    """Jittered, null-bearing pages of the short-page bins (zig-zag simple8b values, RLE / simple8b timestamps,
    <= 1024 rows), with and without GROUP BY series."""
    g = datagen.generate(3000, n_fields=2, n_points=777, value_kind=datagen.I64_WALK, seed=77, jitter_permille=400,
                         jitter_max=999_999, null_page_permille=300, null_row_permille=150)
    pages = engine.upload_pages(g.arena, g.descs)
    w = 60_000_000_000
    fbs, nb = bucket_spec(datagen.TSBS_T0 - 1_000_000, datagen.TSBS_T0 + 776 * datagen.TSBS_STEP + 1_000_000, w)
    sel = np.arange(0, 3000, 3, dtype=np.uint32)
    q = QueryOption([PushedAggregate(c, cabi.TSKV_PT_I64, ALL_AGGS) for c in (1, 2)], series_ids=sel,
                    time_ranges=[(datagen.TSBS_T0 + 7 * datagen.TSBS_STEP, datagen.TSBS_T0 + 700 * datagen.TSBS_STEP)],
                    width=w, first_bucket_start=fbs, n_buckets=nb, group_by_series=gbs)
    assert_results_equal(engine.scan_aggregate(pages, q), orc.scan_aggregate(g.arena, g.descs, q, n_threads=4),
                         what="gbs=%s" % gbs)
    pages.close()


def test_maximum_and_minimum_page_sizes(engine):
    """Column groups are capped at max_datablock_size = 102 400 rows (config/src/tskv/storage_config.rs:136-138);
    the other extreme is a single row. Every codec, decode + scan."""
    rng = np.random.default_rng(102400)
    n = 102_400
    b = datagen.ArenaBuilder()
    ts_reg = datagen.TSBS_T0 + np.arange(n, dtype=np.int64) * 1_000_000
    ts_jit = ts_reg + rng.integers(0, 999, n)
    valid = rng.random(n) > 0.03
    b.add_column_group(1, ts_reg, [(1, cabi.TSKV_PT_I64, np.cumsum(rng.integers(-9, 10, n)), None),
                                   (2, cabi.TSKV_PT_F64, np.cumsum(rng.integers(-2, 3, n)) + rng.random(n), valid),
                                   (3, cabi.TSKV_PT_U64, np.cumsum(rng.integers(0, 3, n)).astype(np.uint64), None)])
    b.add_column_group(2, ts_jit, [(1, cabi.TSKV_PT_I64, rng.integers(-2**62, 2**62, n), valid),      # raw deltas
                                   (2, cabi.TSKV_PT_F64, np.cumsum(rng.integers(-2, 3, n)).astype(np.float64), None),
                                   (3, cabi.TSKV_PT_U64, np.full(n, 7, dtype=np.uint64), None)])         # RLE
    b.add_column_group(3, np.array([datagen.TSBS_T0 + 5]), [(1, cabi.TSKV_PT_I64, np.array([-42]), None),
                                                            (2, cabi.TSKV_PT_F64, np.array([2.5]), None),
                                                            (3, cabi.TSKV_PT_U64, np.array([9], dtype=np.uint64), None)])
    arena, descs = b.finish()
    check_decode(engine, arena, descs)
    pages = engine.upload_pages(arena, descs)
    w = 1_000_000_000
    fbs, nb = bucket_spec(int(ts_reg[0]), int(ts_jit[-1]), w)
    for gbs in (False, True):
        q = make_query(SCAN_FIELDS, time_ranges=[(int(ts_reg[100]), int(ts_reg[-100]))], width=w,
                       first_bucket_start=fbs, n_buckets=nb, group_by_series=gbs)
        assert_results_equal(engine.scan_aggregate(pages, q), orc.scan_aggregate(arena, descs, q, n_threads=3),
                             what="max page gbs=%s" % gbs)
    pages.close()


def test_many_ranges_many_buckets_and_empty_inputs(engine):
    g = datagen.generate(300, n_fields=1, n_points=500, value_kind=datagen.I64_WALK, seed=5, jitter_permille=500, jitter_max=5000)
    pages = engine.upload_pages(g.arena, g.descs)
    t0, step = datagen.TSBS_T0, datagen.TSBS_STEP
    ranges = [(t0 + k * 60 * step, t0 + (k * 60 + 25) * step) for k in range(8)]    # 8 disjoint ranges (the ABI maximum)
    w = 7 * step + 3
    fbs, nb = bucket_spec(t0 - 5000, t0 + 499 * step + 5000, w, origin=11)
    q = make_query([(1, cabi.TSKV_PT_I64)], time_ranges=ranges, origin=11, width=w, first_bucket_start=fbs, n_buckets=nb)
    assert_results_equal(engine.scan_aggregate(pages, q), orc.scan_aggregate(g.arena, g.descs, q), what="8 ranges")
    # overlapping + unsorted ranges behave like their union
    q2 = make_query([(1, cabi.TSKV_PT_I64)], time_ranges=[ranges[3], (ranges[1][0], ranges[2][1]), ranges[1]], origin=11,
                    width=w, first_bucket_start=fbs, n_buckets=nb)
    assert_results_equal(engine.scan_aggregate(pages, q2), orc.scan_aggregate(g.arena, g.descs, q2), what="overlapping ranges")
    # a range that selects nothing / an empty selection list / a column no page has
    for q3 in (make_query([(1, cabi.TSKV_PT_I64)], time_ranges=[(0, 5)]),
               make_query([(1, cabi.TSKV_PT_I64)], series_ids=np.zeros(0, dtype=np.uint32)),
               make_query([(9, cabi.TSKV_PT_F64)])):
        r = engine.scan_aggregate(pages, q3)
        assert_results_equal(r, orc.scan_aggregate(g.arena, g.descs, q3), what="empty")
        assert r.validity[1:].sum() == 0 and r.values[0].sum() == 0
    pages.close()
    # an arena without pages
    empty = engine.upload_pages(np.zeros(0, dtype=np.uint8), np.zeros(0, dtype=cabi.PAGE_DESC_DTYPE))
    r = engine.scan_aggregate(empty, make_query([(1, cabi.TSKV_PT_I64)]))
    assert r.column(1, "count")[0][0, 0] == 0
    empty.close()


def test_host_resident_pages_verify_crc_on_every_read(engine):
    """HOST_RESIDENT | VERIFY_CRC: the device re-checks the CRC32 of every page a scan pulls over PCIe
    (Page::crc_validation on each read, tsm/reader.rs:259). Corruption after the upload is caught by the next scan."""
    g = datagen.generate(400, n_fields=2, n_points=300, value_kind=datagen.MIXED, seed=12, jitter_permille=300, jitter_max=999)
    arena = g.arena.copy()
    q = QueryOption([PushedAggregate(1, cabi.TSKV_PT_I64, ["count", "sum"]), PushedAggregate(3, cabi.TSKV_PT_F64, ["count", "max"])],
                    series_ids=np.arange(0, 400, 2, dtype=np.uint32).repeat(1)[:150])
    hp = engine.upload_pages(arena, g.descs, verify_crc=True, host_resident=True)
    assert_results_equal(engine.scan_aggregate(hp, q), orc.scan_aggregate(arena, g.descs, q), what="host-resident verified")
    victim = next(i for i, d in enumerate(g.descs) if d["phys_type"] == cabi.TSKV_PT_I64 and d["series_id"] == 4 and d["column_id"] == 1)
    arena[int(g.descs[victim]["offset"]) + int(g.descs[victim]["size"]) - 3] ^= 0x21
    with pytest.raises(TskvError) as e:
        engine.scan_aggregate(hp, q)
    assert e.value.status == cabi.TSKV_ERR_CRC_MISMATCH and e.value.page == victim
    # pages of series that are not selected are not read, so their corruption goes unnoticed (like the reference)
    arena[int(g.descs[victim]["offset"]) + int(g.descs[victim]["size"]) - 3] ^= 0x21
    other = next(i for i, d in enumerate(g.descs) if d["series_id"] == 399 and d["phys_type"] != cabi.TSKV_PT_TIME)
    arena[int(g.descs[other]["offset"]) + 40] ^= 0xff
    engine.scan_aggregate(hp, q)
    hp.close()


def test_host_resident_series_with_fields_in_different_bins(engine):
    """A series whose selected fields decode in different kind bins (i64 simple8b + f64 gorilla): every bin's gather has
    to bring the column group's time page itself - the bins run on different streams (round-1 advisor finding). Also
    decode-only on a host-resident page set, which must read the mapped host arena, not the scans' gather target."""
    rng = np.random.default_rng(77)
    arena, descs, _ = random_arena(rng, n_series=300, n_points=257, fields=((1, cabi.TSKV_PT_I64), (2, cabi.TSKV_PT_F64)),
                                   jitter=200, null_frac=0.02)
    t_lo, t_hi = 1_000_000 - 400, 1_000_000 + 300_000
    fbs, nb = bucket_spec(t_lo, t_hi, 17_000, origin=3)
    q = make_query(((1, cabi.TSKV_PT_I64), (2, cabi.TSKV_PT_F64)), aggs=("count", "sum", "min", "max", "mean"),
                   series_ids=np.arange(0, 300, 3, dtype=np.uint32), origin=3, width=17_000, first_bucket_start=fbs,
                   n_buckets=nb)
    exp = orc.scan_aggregate(arena, descs, q)
    for verify in (True, False):
        for _ in range(3):  # fresh page sets: the gather target starts out uninitialised
            hp = engine.upload_pages(arena, descs, verify_crc=verify, host_resident=True)
            assert_results_equal(engine.scan_aggregate(hp, q), exp, what="host-resident, two bins per series")
            hp.close()
    hp = engine.upload_pages(arena, descs, verify_crc=True, host_resident=True)
    got = engine.decode_pages(hp, descs, 0, 60)
    exp_pages = orc.decode_pages(arena, descs, 0, 60)
    for (gv, gm), (ev, em) in zip(got, exp_pages):
        assert (gm == em).all() and (gv[em] == ev[em]).all()
    hp.close()


def test_two_shard_unbucketed_first_last_with_different_time_minima(engine):
    """Unbucketed FIRST/LAST across series merged from two shards whose arenas start at different times: the tie-break
    keys must be built from the query alone (TSKV_QUERY_MULTI_RANK), not from each rank's own time bounds
    (round-1 advisor finding); and a multi-rank scan without the global series list is refused."""
    import torch
    from cnosdb_b200.parallel import device_tensor
    rng = np.random.default_rng(5)
    fields = ((1, cabi.TSKV_PT_I64), (2, cabi.TSKV_PT_F64))
    parts = [random_arena(rng, n_series=20, n_points=200, fields=fields, ids=range(0, 20), t0=5_000_000),
             random_arena(rng, n_series=20, n_points=200, fields=fields, ids=range(20, 40), t0=1_000_000)]
    b = datagen.ArenaBuilder()
    for _, _, truth in parts:
        for sid, cgs in truth.items():
            for ts, cols in cgs:
                b.add_column_group(sid, ts, [(c, pt, cols[c][0], cols[c][1], None) for c, pt in fields])
    arena, descs = b.finish()
    sel = np.arange(1, 40, 2, dtype=np.uint32)
    q = make_query(fields, series_ids=sel, time_ranges=[(900_000, 6_000_000)], multi_rank=True)
    exp = orc.scan_aggregate(arena, descs, q)
    dev = torch.device("cuda", engine.device)
    scans, regions, keep = [], [], []
    for a, d, _ in parts:
        pages = engine.upload_pages(a, d)
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
        assert_results_equal(s.finalize(), exp, what="2-shard unbucketed first/last")
        s.close()
    with pytest.raises(TskvError) as e:
        engine.prepare(keep[0], make_query(fields, time_ranges=[(900_000, 6_000_000)], multi_rank=True))
    assert e.value.status == cabi.TSKV_ERR_INVALID_ARG
    for pages in keep:
        pages.close()


def test_statistics_pruning_skips_column_groups_outside_the_time_ranges(engine):
    """filter_column_groups on the device (reader/chunk.rs:12-50): a page set uploaded once and scanned with a narrow time
    range reads only the column groups whose time bounds overlap it - same results, fewer pages (page_read_count /
    page_read_bytes / pruned_page_count) - with bounds computed by the library or handed in like ColumnGroup::time_range()."""
    rng = np.random.default_rng(21)
    fields = ((1, cabi.TSKV_PT_I64), (2, cabi.TSKV_PT_F64))
    arena, descs, truth = random_arena(rng, n_series=120, n_points=200, fields=fields, multi_cg=True, null_frac=0.05)
    groups = [(sid, ts) for sid, cgs in truth.items() for ts, _ in cgs]   # descriptor order: series by series, group by group
    lo, hi = 1_000_000 + 150_000, 1_000_000 + 180_000
    ranges = [(lo, hi), (1_000_000 - 50, 1_000_000 + 10)]
    q = make_query(fields, aggs=("count", "sum", "min", "max", "mean"), time_ranges=ranges, group_by_series=True)
    exp = orc.scan_aggregate(arena, descs, q)
    overlapping = sum(1 for _, ts in groups if any(ts.min() <= b and ts.max() >= a for a, b in ranges))
    assert 0 < overlapping < len(groups)
    for given in (False, True):
        pages = engine.upload_pages(arena, descs)
        if given:
            pages.set_time_bounds([(int(ts.min()), int(ts.max())) for _, ts in groups])
        assert_results_equal(engine.scan_aggregate(pages, q), exp, what="pruned scan (bounds given: %s)" % given)
        c = engine.counters()
        assert c["page_read_count"] == 3 * overlapping, (c["page_read_count"], overlapping)
        assert c["pruned_page_count"] == 2 * (len(groups) - overlapping)
        all_time = make_query(fields, aggs=("count",), group_by_series=True)   # no ranges: nothing is pruned
        engine.scan_aggregate(pages, all_time)
        c = engine.counters()
        assert c["page_read_count"] == 3 * len(groups) and c["pruned_page_count"] == 0
        pages.close()
    with pytest.raises(TskvError):
        p2 = engine.upload_pages(arena, descs)
        try:
            p2.set_time_bounds([(0, 1)])   # wrong number of column groups
        finally:
            p2.close()


@pytest.mark.parametrize("variant", ["plain", "nulls", "jitter", "multi_cg"])
def test_field_predicates_filter_rows_like_the_reference_data_filter(engine, variant):
    """`column <op> constant` row filters pushed into the scan (DataFilter, reader/filter.rs:23-142): a row survives only
    if every comparison is TRUE (NULL drops it), for all projected columns, counts and first()/last() included."""
    rng = np.random.default_rng(300 + len(variant))
    fields = ((1, cabi.TSKV_PT_I64), (2, cabi.TSKV_PT_F64), (3, cabi.TSKV_PT_U64))
    kw = dict(n_series=90, n_points=300, fields=fields)
    if variant == "nulls":
        kw["null_frac"] = 0.15
    if variant == "jitter":
        kw.update(jitter=300, null_frac=0.03)
    if variant == "multi_cg":
        kw.update(multi_cg=True, null_frac=0.05)
    arena, descs, _ = random_arena(rng, **kw)
    pages = engine.upload_pages(arena, descs)
    t_lo, t_hi = 1_000_000 - 400, 1_000_000 + 700_000
    fbs, nb = bucket_spec(t_lo, t_hi, 17_000, origin=3)
    proj = fields[:2]
    cases = [
        [(1, cabi.TSKV_PT_I64, ">", 0)],
        [(2, cabi.TSKV_PT_F64, "<=", 1.5), (1, cabi.TSKV_PT_I64, "!=", 7)],
        [(3, cabi.TSKV_PT_U64, ">=", 2**63 + 40)],                          # a column that is not projected
        [(9, cabi.TSKV_PT_I64, "==", 1)],                                   # a column no group holds: no row survives
        [(1, cabi.TSKV_PT_I64, "<", -10**9)],                               # nothing passes
    ]
    for preds in cases:
        for group_by_series in (False, True):
            for ranges in ([], [(t_lo + 30_000, t_lo + 250_000)]):
                q = make_query(proj, time_ranges=ranges, origin=3, width=17_000, first_bucket_start=fbs, n_buckets=nb,
                               group_by_series=group_by_series, predicates=preds)
                got = engine.scan_aggregate(pages, q)
                exp = orc.scan_aggregate(arena, descs, q)
                assert_results_equal(got, exp, what="predicates %s gbs=%s %s %s" % (preds, group_by_series, ranges, variant))
        q = make_query(proj, aggs=("count", "sum", "min", "max", "mean"), predicates=preds)   # unbucketed, staged flush
        assert_results_equal(engine.scan_aggregate(pages, q), orc.scan_aggregate(arena, descs, q), what="predicates unbucketed")
    hp = engine.upload_pages(arena, descs, verify_crc=True, host_resident=True)
    q = make_query(proj, width=17_000, origin=3, first_bucket_start=fbs, n_buckets=nb, predicates=cases[1])
    assert_results_equal(engine.scan_aggregate(hp, q), orc.scan_aggregate(arena, descs, q), what="predicates, host-resident pages")
    with pytest.raises(TskvError):
        engine.scan_aggregate(pages, make_query(proj, predicates=[(1, cabi.TSKV_PT_F64, ">", 0.0)]))  # wrong column type
    hp.close()
    pages.close()


def random_tombstones(rng, descs, t_lo, t_hi, n=60):
    """Column masks, series-scoped row drops and a few page-set-wide row drops over random sub-ranges."""
    fields = descs[descs["phys_type"] != cabi.TSKV_PT_TIME]
    out = []
    for _ in range(n):
        d = fields[int(rng.integers(0, len(fields)))]
        a = int(rng.integers(t_lo, t_hi))
        b = a + int(rng.integers(0, (t_hi - t_lo) // 6))
        kind = rng.random()
        if kind < 0.6:
            out.append((int(d["series_id"]), int(d["column_id"]), a, b))
        elif kind < 0.9:
            out.append((int(d["series_id"]), None, a, b))
        else:
            out.append((None, None, a, a + (b - a) // 8))
    out.append((int(fields[0]["series_id"]), int(fields[0]["column_id"]), t_hi, t_lo))  # empty range: ignored
    return cabi.tombstones(out)


@pytest.mark.parametrize("variant", ["plain", "nulls", "jitter", "multi_cg", "raw"])
def test_scan_with_tombstones_matches_decode_pages_semantics(engine, variant):
    """TsmTombstone ranges through the fused scan (tsm/reader.rs:507-551): dropped rows, nulled column values, and
    the first()/last() consequences, against the oracle's binary-search restatement."""
    rng = np.random.default_rng(1000 + len(variant))
    kw = dict(n_series=70, n_points=333, fields=SCAN_FIELDS)
    if variant == "nulls":
        kw["null_frac"] = 0.2
    if variant == "jitter":
        kw["jitter"] = 300
    if variant == "multi_cg":
        kw.update(multi_cg=True, null_frac=0.05)
    if variant == "raw":
        kw["raw_frac"] = 0.5
    arena, descs, _ = random_arena(rng, **kw)
    pages = engine.upload_pages(arena, descs)
    t_lo, t_hi = 1_000_000 - 400, 1_000_000 + 700_000
    tombs = random_tombstones(rng, descs, t_lo, 1_000_000 + 340_000)
    pages.set_tombstones(tombs)
    fbs, nb = bucket_spec(t_lo, t_hi, 17_000, origin=3)
    sel = np.array(sorted(rng.choice(np.arange(80), 45, replace=False)), dtype=np.uint32)
    for group_by_series in (False, True):
        for series_ids in (sel, None):
            for ranges in ([(t_lo + 30_000, t_lo + 250_000)], []):
                q = make_query(SCAN_FIELDS, series_ids=series_ids, time_ranges=ranges, origin=3, width=17_000,
                               first_bucket_start=fbs, n_buckets=nb, group_by_series=group_by_series)
                got = engine.scan_aggregate(pages, q)
                exp = orc.scan_aggregate(arena, descs, q, tombstones=tombs)
                assert_results_equal(got, exp, what="tomb %s gbs=%s %s" % (variant, group_by_series, ranges))
        q = make_query(SCAN_FIELDS, series_ids=sel, group_by_series=group_by_series)  # unbucketed
        assert_results_equal(engine.scan_aggregate(pages, q), orc.scan_aggregate(arena, descs, q, tombstones=tombs), what="tomb unbucketed")
    q_plain = make_query(SCAN_FIELDS, aggs=("count", "sum"), series_ids=sel)
    with_t = engine.scan_aggregate(pages, q_plain)
    pages.set_tombstones([])  # cleared: back to the plain result
    without = engine.scan_aggregate(pages, q_plain)
    assert_results_equal(without, orc.scan_aggregate(arena, descs, q_plain), what="tombstones cleared")
    assert int(with_t.column(1, "count")[0].sum()) < int(without.column(1, "count")[0].sum())
    pages.close()


def test_tombstones_golden_generic_time_pages_and_api_rules(engine):
    b = datagen.ArenaBuilder()
    for ts, vals in (([1], [111]), ([2, 3, 4], [212, 213, 214]), ([4, 5, 6], [314, 315, 316]), ([8, 9], [418, 419])):
        b.add_column_group(1, np.array(ts, dtype=np.int64), [(1, cabi.TSKV_PT_I64, np.array(vals, dtype=np.int64), None)])
    # a raw-encoded time page (one delta > 2^60 - 1) goes through the row-wise kernel
    ts = np.concatenate([-(2**62) + np.arange(40, dtype=np.int64) * 1000, [2**61]]).astype(np.int64)
    b.add_column_group(2, ts, [(1, cabi.TSKV_PT_I64, np.arange(41, dtype=np.int64), None),
                               (2, cabi.TSKV_PT_F64, np.arange(41, dtype=np.float64), None)])
    arena, descs = b.finish()
    pages = engine.upload_pages(arena, descs)
    q = make_query([(1, cabi.TSKV_PT_I64)], series_ids=np.array([1], dtype=np.uint32))
    prepared = engine.prepare(pages, q)
    tombs = cabi.tombstones([(1, 1, 2, 6), (2, 1, -(2**62) + 5000, -(2**62) + 9000), (2, None, 2**61, 2**61),
                             (None, None, -(2**62), -(2**62) + 1500)])
    pages.set_tombstones(tombs)
    with pytest.raises(TskvError) as e:  # prepared before the change: refused, not silently stale
        prepared.run()
    assert e.value.status == cabi.TSKV_ERR_INVALID_ARG
    prepared.close()
    got = engine.scan_aggregate(pages, q)  # compact_test.rs:421-521: [111, None x5, 418, 419]
    assert int(got.column(1, "count")[0][0, 0]) == 3 and int(got.column(1, "sum")[0][0, 0].view(np.int64)) == 948
    q2 = make_query([(1, cabi.TSKV_PT_I64), (2, cabi.TSKV_PT_F64)], group_by_series=True)
    got, exp = engine.scan_aggregate(pages, q2), orc.scan_aggregate(arena, descs, q2, tombstones=tombs)
    assert_results_equal(got, exp, what="raw time page + tombstones")
    assert int(got.column(1, "count")[0][1, 0]) == 41 - 5 - 1 - 2 and int(got.column(2, "count")[0][1, 0]) == 41 - 1 - 2
    with pytest.raises(TskvError) as e:
        pages.set_tombstones(cabi.tombstones([(None, 1, 0, 10)]))
    assert e.value.status == cabi.TSKV_ERR_INVALID_ARG
    pages.close()


@pytest.mark.parametrize("seed", [6, 9, 37])
def test_gorilla_mixed_pages_agree_with_oracle(engine, seed):
    """Gorilla pages of mixed values (jittered, with nulls, <= 1024 rows: the short-page bins) against the oracle."""
    g = datagen.generate(1500, n_fields=2, n_points=1000, value_kind=datagen.MIXED, seed=seed, jitter_permille=300,
                         jitter_max=999_999, null_page_permille=300, null_row_permille=120)
    pages = engine.upload_pages(g.arena, g.descs)
    w = 60_000_000_000
    fbs, nb = bucket_spec(datagen.TSBS_T0 - 1_000_000, datagen.TSBS_T0 + 999 * datagen.TSBS_STEP + 1_000_000, w)
    sel = np.arange(0, 1500, 2, dtype=np.uint32)
    cols = [PushedAggregate(1, cabi.TSKV_PT_I64, ALL_AGGS), PushedAggregate(3, cabi.TSKV_PT_F64, ALL_AGGS),
            PushedAggregate(4, cabi.TSKV_PT_F64, ("count", "sum", "first"))]
    for gbs in (False, True):
        q = QueryOption(cols, series_ids=sel, time_ranges=[(datagen.TSBS_T0 + 7 * datagen.TSBS_STEP, datagen.TSBS_T0 + 900 * datagen.TSBS_STEP)],
                        width=w, first_bucket_start=fbs, n_buckets=nb, group_by_series=gbs)
        assert_results_equal(engine.scan_aggregate(pages, q), orc.scan_aggregate(g.arena, g.descs, q, n_threads=4),
                             what="gorilla seed=%d gbs=%s" % (seed, gbs))
    pages.close()


@pytest.mark.parametrize("case,status", [("extra_values", 0), ("early_sentinel", cabi.TSKV_ERR_BITSET_MISMATCH),
                                         ("truncated", cabi.TSKV_ERR_SHORT_BLOCK), ("sentinel_valued_data", 0),
                                         ("first_value_only", cabi.TSKV_ERR_SHORT_BLOCK)])
@pytest.mark.parametrize("jitter", [False, True])
def test_gorilla_stream_end_cases(engine, case, status, jitter):
    """The end of a gorilla stream (float.rs:480-591): more values than valid rows are decoded and ignored, a
    sentinel before the bitset is served is a mismatch, a stream without sentinel is an unexpected end of block.
    Regular timestamps make a run-length time page, jittered ones a simple8b time page: the two time classes of the
    short Gorilla bins."""
    n = 200
    vals = np.cumsum(np.arange(n) % 5).astype(np.float64) * 0.37 + 1.5
    ts = datagen.TSBS_T0 + np.arange(n, dtype=np.int64) * datagen.TSBS_STEP
    if jitter:
        ts += np.random.default_rng(11).integers(0, datagen.TSBS_STEP // 2, n)
    b = datagen.ArenaBuilder()
    b.add_page(datagen.build_page(datagen.encode_timestamps(ts), n), 5, 0, cabi.TSKV_PT_TIME, n)
    if case == "extra_values":    # 230 encoded values for 200 rows
        data = datagen.encode_floats(np.concatenate([vals, np.arange(30) * 3.25]))
    elif case == "early_sentinel":  # 150 encoded values for 200 valid rows
        data = datagen.encode_floats(vals[:150])
    elif case == "truncated":     # cut inside the stream: no sentinel
        data = datagen.encode_floats(vals)[:-24]
    elif case == "sentinel_valued_data":  # the first value and "repeat" elements are pushed without a sentinel test
        # the encoder refuses the sentinel (float.rs:58), so the stream is written by hand: first = sentinel, 6 x "repeat",
        # one full-width element giving 2.5, the terminator; 8 rows
        sent, v25 = 0x7FF80000000000FF, int(np.float64(2.5).view(np.uint64))
        bits = "0" * 6 + "11" + "00000" + "000000" + format(sent ^ v25, "064b") + "11" + "00000" + "000000" + format(v25 ^ sent, "064b")
        data = np.frombuffer(bytes([6, 0x10]) + sent.to_bytes(8, "big") + int(bits, 2).to_bytes(len(bits) // 8, "big"), dtype=np.uint8)
        n = 8
        ts = ts[:n]
        b = datagen.ArenaBuilder()
        b.add_page(datagen.build_page(datagen.encode_timestamps(ts), n), 5, 0, cabi.TSKV_PT_TIME, n)
    else:                         # nothing after the first value: refill_cache fails (float.rs:447-466)
        data = np.frombuffer(bytes([6, 0x10]) + (0x7FF80000000000FF).to_bytes(8, "big"), dtype=np.uint8)
    b.add_page(datagen.build_page(data, n), 5, 1, cabi.TSKV_PT_F64, n)
    b.add_column_group(6, ts, [(1, cabi.TSKV_PT_F64, np.arange(n) * 0.5, None)])
    arena, descs = b.finish()
    assert time_page_is_rle(arena, descs[0]) != jitter
    aggs = ("count", "first", "last") if case == "sentinel_valued_data" else ALL_AGGS  # (no NaN into sum/min/max)
    q = QueryOption([PushedAggregate(1, cabi.TSKV_PT_F64, aggs)], group_by_series=True,
                    time_ranges=[(int(ts[0]), int(ts[6]))] if case == "sentinel_valued_data" else [])
    pages = engine.upload_pages(arena, descs)
    if status == 0:
        assert_results_equal(engine.scan_aggregate(pages, q), orc.scan_aggregate(arena, descs, q), what=case)
    else:
        with pytest.raises(orc.OracleError) as oe:
            orc.scan_aggregate(arena, descs, q)
        assert oe.value.status == status
        with pytest.raises(TskvError) as ge:
            engine.scan_aggregate(pages, q)
        assert ge.value.status == status and ge.value.page == 1
    pages.close()
