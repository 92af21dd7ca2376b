"""The fused scan's lockstep schedule (simple8b time pages, GROUP BY bucket / tags / edges / labels, no FIRST / LAST). A
warp whose 32 pages start and end at the same row, in one bucket or the next, walks one bucket schedule for all of them
while every lane compares its own timestamps; a row outside the next bucket hands the warp to the segment loop.

One page set holds a block of 32 series (one chunk per query column) for each case:
- jitter of +-1 around a grid whose rows fall on the bucket edges: edge rows on both sides of an edge in different lanes,
- a gap wider than the bucket in half of the lanes partway through the page (the handoff),
- a gap in every lane: buckets that no lane has a row in,
- another start bucket or another length in some lanes (the segment loop from the start),
- NULLs in every page (sparse bitmap words; with the field predicate, sparse keep words too),
- jitter of almost half a step,
and a tail chunk with lanes that hold no page (the segment loop). It is scanned with pages whole and cut into parts,
with and without a time range that starts and ends inside buckets, against the oracle (COUNT / integer SUM / MIN / MAX
bit for bit, f64 within 1e-6) and its points counter; with tombstones; and with edges, labels and GROUP BY tags against
the exact reference. Rows past the last bucket report TSKV_ERR_BUCKET_RANGE as the oracle does."""
import numpy as np
import pytest

from cnosdb_b200 import cabi, datagen
from cnosdb_b200.engine import TskvError
from oracle import pyoracle as orc
from tests.edges_reference import exact_aggregate_edges
from tests.group_reference import exact_aggregate_grouped
from tests.helpers import assert_matches_exact, assert_results_equal, bucket_spec, make_query, time_page_is_rle
from tests.labels_reference import exact_aggregate_labels

pytestmark = pytest.mark.gpu

FIELDS = ((1, cabi.TSKV_PT_I64), (2, cabi.TSKV_PT_F64))  # simple8b i64 and Gorilla f64 values: one bin each
AGGS = ("count", "sum", "min", "max", "mean")  # FIRST / LAST take the segment loop
T0, STEP, W = 1_200_000, 1000, 6000  # 6-row buckets; every 6th grid point lies on a bucket edge, as in C4
N = 700
CASES = ("jitter", "gap", "empty", "unaligned", "nulls", "wide_jitter")
N_SERIES = 32 * len(CASES) + 10  # + a tail chunk of 10 pages per bin
RANGES = ([], [(T0 + 130_500, T0 + 555_250)])


def series_rows(rng, sid):
    """(timestamps, valid mask or None) of series sid."""
    case = CASES[sid // 32] if sid < 32 * len(CASES) else "jitter"
    n, t0, jit, valid = N, T0, 1, None
    keep = np.ones(N, dtype=bool)
    if case == "gap" and sid % 2:
        keep[300 + sid % 5:320] = False  # 14-18 missing rows: more than two buckets
    elif case == "empty":
        keep[400:413] = False
    elif case == "unaligned" and sid % 4 == 1:
        t0 = T0 + 2 * STEP
    elif case == "unaligned" and sid % 4 == 2:
        n, keep = 650, keep[:650]
    elif case == "nulls":
        valid = rng.random(n) >= 0.3
    elif case == "wide_jitter":
        jit = STEP // 2 - 1
    ts = t0 + np.arange(n, dtype=np.int64) * STEP + rng.integers(-jit, jit + 1, n)
    return ts[keep], (None if valid is None else valid[keep])


def make_arena(seed):
    rng = np.random.default_rng(seed)
    b = datagen.ArenaBuilder()
    truth = {}
    for sid in range(N_SERIES):
        ts, valid = series_rows(rng, sid)
        n = ts.size
        fl, cols = [], {}
        for col, pt in FIELDS:
            if pt == cabi.TSKV_PT_F64:
                vals = np.cumsum(rng.integers(-3, 4, n)).astype(np.float64) + rng.random(n)
            else:
                vals = np.cumsum(rng.integers(-50, 51, n)).astype(np.int64)
            fl.append((col, pt, vals, valid, None))
            cols[col] = (vals, np.ones(n, dtype=bool) if valid is None else valid)
        b.add_column_group(sid, ts, fl)
        truth[sid] = [(ts, cols)]
    arena, descs = b.finish()
    return arena, descs, truth


@pytest.fixture(scope="module")
def arena():
    return make_arena(17)


def grid():
    fbs, nb = bucket_spec(T0 - STEP, T0 + (N + 3) * STEP, W)
    return dict(width=W, first_bucket_start=fbs, n_buckets=nb)


def time_pages_are_s8b(arena_, descs):
    # (a jittered time page is simple8b-coded: the test must reach the simple8b-timestamp bins)
    return not any(time_page_is_rle(arena_, d) for d in descs if d["column_id"] == 0)


@pytest.mark.parametrize("parts", ["1", "3"])
@pytest.mark.parametrize("pred", [False, True])
def test_lockstep_matches_oracle(engine, arena, parts, pred, monkeypatch):
    monkeypatch.setenv("TSKV_PARTS", parts)
    a, descs, _ = arena
    assert time_pages_are_s8b(a, descs)
    pages = engine.upload_pages(a, descs)
    sel = np.arange(N_SERIES, dtype=np.uint32)
    preds = [(1, cabi.TSKV_PT_I64, ">", -20)] if pred else []
    for ranges in RANGES:
        q = make_query(FIELDS, AGGS, series_ids=sel, time_ranges=ranges, predicates=preds, **grid())
        got = engine.scan_aggregate(pages, q)
        exp, pts = orc.scan_aggregate(a, descs, q, return_points=True)
        what = "parts=%s pred=%s ranges=%s" % (parts, pred, ranges)
        assert_results_equal(got, exp, what=what)
        assert engine.counters()["points_decoded"] == pts, what
        again = engine.scan_aggregate(pages, q)  # integer cells do not depend on the order of the table updates
        for j, (col, agg) in enumerate(got.names):
            if got.phys[col] != cabi.TSKV_PT_F64 and agg != "mean":
                assert (again.values[j] == got.values[j]).all(), what
    pages.close()


@pytest.mark.parametrize("parts", ["1", "3"])
def test_lockstep_with_tombstones(engine, arena, parts, monkeypatch):
    """Tombstones keep the whole scan on the segment loop."""
    monkeypatch.setenv("TSKV_PARTS", parts)
    a, descs, _ = arena
    pages = engine.upload_pages(a, descs)
    tombs = cabi.tombstones([(5, None, T0 + 100_000, T0 + 140_000), (40, 1, T0 + 10_000, T0 + 300_500),
                             (None, None, T0 + 600_000, T0 + 601_000)])
    pages.set_tombstones(tombs)
    q = make_query(FIELDS, AGGS, series_ids=np.arange(N_SERIES, dtype=np.uint32), **grid())
    exp = orc.scan_aggregate(a, descs, q, tombstones=tombs)
    assert_results_equal(engine.scan_aggregate(pages, q), exp, what="tombstones parts=%s" % parts)
    pages.close()


def edges_and_labels():
    """Irregular edges (a few bucket widths, some edges on grid rows) and labels folding them onto 5 outputs."""
    e = [T0 - STEP]
    widths = (6000, 4000, 9000, 6000, 1500, 6000, 12000)
    i = 0
    while e[-1] <= T0 + (N + 3) * STEP:
        e.append(e[-1] + widths[i % len(widths)])
        i += 1
    e = np.array(e, dtype=np.int64)
    labels = (np.arange(e.size - 1) % 5).astype(np.uint32)
    return e, labels


def edge_query(ranges):
    e, _ = edges_and_labels()
    return make_query(FIELDS, AGGS, series_ids=np.arange(N_SERIES, dtype=np.uint32), time_ranges=ranges,
                      n_buckets=e.size - 1)


@pytest.mark.parametrize("parts", ["1", "3"])
def test_lockstep_edges_labels_and_tags(engine, arena, parts, monkeypatch):
    monkeypatch.setenv("TSKV_PARTS", parts)
    a, descs, truth = arena
    pages = engine.upload_pages(a, descs)
    e, labels = edges_and_labels()
    for ranges in RANGES:
        what = "parts=%s ranges=%s" % (parts, ranges)
        q = edge_query(ranges)
        assert_matches_exact(engine.scan_aggregate(pages, q, edges=e), exact_aggregate_edges(truth, q, e),
                             what="edges " + what, first_last=False)
        ql = make_query(FIELDS, AGGS, series_ids=q.series_ids, time_ranges=ranges, n_buckets=5)
        assert_matches_exact(engine.scan_aggregate(pages, ql, edges=e, labels=labels),
                             exact_aggregate_labels(truth, ql, e, labels), what="labels " + what, first_last=False)
        # GROUP BY tags: groups of 8 neighbouring series (4 per chunk) and one group that spans chunks
        gq = make_query(FIELDS, AGGS, series_ids=q.series_ids, time_ranges=ranges, **grid())
        gids = (np.arange(N_SERIES) // 8).astype(np.uint32)
        gids[N_SERIES - 30:] = 3
        ng = int(gids.max()) + 1
        assert_matches_exact(engine.scan_aggregate(pages, gq, group_ids=gids, n_groups=ng),
                             exact_aggregate_grouped(truth, gq, gids, ng), what="tags " + what, first_last=False)
    pages.close()


@pytest.mark.parametrize("parts", ["1", "3"])
def test_rows_past_the_last_bucket(engine, arena, parts, monkeypatch):
    """The schedule hands off at the last bucket, and the segment loop reports TSKV_ERR_BUCKET_RANGE as the oracle does."""
    monkeypatch.setenv("TSKV_PARTS", parts)
    a, descs, _ = arena
    pages = engine.upload_pages(a, descs)
    fbs, nb = bucket_spec(T0 - STEP, T0 + 500 * STEP, W)
    q = make_query(FIELDS, AGGS, series_ids=np.arange(N_SERIES, dtype=np.uint32), width=W, first_bucket_start=fbs,
                   n_buckets=nb)
    with pytest.raises(orc.OracleError) as oe:
        orc.scan_aggregate(a, descs, q)
    assert oe.value.status == cabi.TSKV_ERR_BUCKET_RANGE
    with pytest.raises(TskvError) as ge:
        engine.scan_aggregate(pages, q)
    assert ge.value.status == cabi.TSKV_ERR_BUCKET_RANGE
    pages.close()
