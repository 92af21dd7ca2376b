"""The fused scan's uniform bucket schedule (RLE time pages, GROUP BY bucket, no FIRST / LAST). A warp whose pages all
start at the same row and time and end at the same row walks one bucket schedule for all of them; any other warp keeps
the per-lane segment loop. The aligned page set runs every chunk on the uniform schedule: pages with nulls, a range
that cuts buckets, a tail chunk with idle lanes, pages cut into parts. The mixed page set adds one block of 32 series
with another start time or another length: the chunks that hold them take the segment loop, the others the uniform
schedule."""
import numpy as np
import pytest

from cnosdb_b200 import cabi, datagen
from cnosdb_b200.engine import TskvError
from oracle import pyoracle as orc
from tests.helpers import assert_results_equal, bucket_spec, make_query

pytestmark = pytest.mark.gpu

# one query column per bin (simple8b i64 / Gorilla f64), so a bin's tail chunk holds pages of one column only
FIELDS = ((1, cabi.TSKV_PT_I64), (2, cabi.TSKV_PT_F64))
AGGS = ("count", "sum", "min", "max", "mean")  # FIRST / LAST take the segment loop
T0, STEP, W = 1_000_000, 1000, 6000  # 6-row buckets, like C4's 10 s rows in 1-minute buckets
N_SERIES = 150  # 4 full chunks of 32 pages per bin and a tail chunk of 22
ODD = range(64, 96)  # the mixed set's block: another start time (odd ids) or another length (even ids)


def make_arena(rng, n_series, odd=()):
    b = datagen.ArenaBuilder()
    for sid in range(n_series):
        n, t0 = 700, T0
        if sid in odd:
            if sid % 2:
                t0 = T0 + 2 * STEP  # another bucket phase
            else:
                n = 650 if sid % 4 == 0 else 100  # the last part ends elsewhere, or the page is never cut
        ts = t0 + np.arange(n, dtype=np.int64) * STEP
        nulls = sid % 13 == 6
        fl = []
        for col, pt in FIELDS:
            valid = rng.random(n) >= 0.3 if nulls else None
            if pt == cabi.TSKV_PT_F64:
                vals = np.cumsum(rng.integers(-3, 4, n)).astype(np.float64) + rng.random(n)
            else:
                vals = np.cumsum(rng.integers(-50, 51, n)).astype(np.int64)
            fl.append((col, pt, vals, valid, None))
        b.add_column_group(sid, ts, fl)
    return b.finish()


@pytest.mark.parametrize("parts", ["1", "3"])
@pytest.mark.parametrize("layout", ["aligned", "mixed"])
def test_uniform_schedule_matches_oracle(engine, layout, parts, monkeypatch):
    monkeypatch.setenv("TSKV_PARTS", parts)
    rng = np.random.default_rng(91)
    arena, descs = make_arena(rng, N_SERIES, ODD if layout == "mixed" else ())
    pages = engine.upload_pages(arena, descs)
    fbs, nb = bucket_spec(T0 - W, T0 + 800 * STEP, W)
    sel = np.arange(N_SERIES, dtype=np.uint32)
    # no range, and one that starts and ends inside a bucket (rows 131 and 555; buckets start at rows 2 mod 6)
    for ranges in ([], [(T0 + 130_500, T0 + 555_250)]):
        q = make_query(FIELDS, AGGS, series_ids=sel, time_ranges=ranges, width=W, first_bucket_start=fbs, n_buckets=nb)
        got = engine.scan_aggregate(pages, q)
        exp, pts = orc.scan_aggregate(arena, descs, q, return_points=True)
        assert_results_equal(got, exp, what="%s parts=%s ranges=%s" % (layout, parts, ranges))
        assert engine.counters()["points_decoded"] == pts
    pages.close()


@pytest.mark.parametrize("parts", ["1", "3"])
def test_bucket_range_error_on_the_uniform_schedule(engine, parts, monkeypatch):
    """Rows past the last bucket: the uniform schedule reports TSKV_ERR_BUCKET_RANGE where a bucket starts, like the
    segment loop and the oracle (without FIRST / LAST, so the scan does not take the SEL kernel)."""
    monkeypatch.setenv("TSKV_PARTS", parts)
    arena, descs = make_arena(np.random.default_rng(5), 40)
    pages = engine.upload_pages(arena, descs)
    fbs, nb = bucket_spec(T0 - W, T0 + 100 * STEP, W)
    q = make_query(FIELDS, AGGS, width=W, first_bucket_start=fbs, n_buckets=nb)
    with pytest.raises(orc.OracleError) as oe:
        orc.scan_aggregate(arena, descs, q)
    assert oe.value.status == cabi.TSKV_ERR_BUCKET_RANGE
    with pytest.raises(TskvError) as e:
        engine.scan_aggregate(pages, q)
    assert e.value.status == cabi.TSKV_ERR_BUCKET_RANGE
    pages.close()
