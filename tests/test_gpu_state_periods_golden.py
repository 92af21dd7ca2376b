"""The reference's state_at / duration_in answers with a start time (tests/golden/state_agg_periods_slt.json) through the
scan and engine.state_at / engine.duration_in: state_at.slt and duration_in.slt over their states table (string states
coded to i64), the StatePeriods unit fixture of state_agg_data.rs (joined), and the compact-agg errors: of the compact
aggregate, and of a state_agg over a cell of one row."""
import numpy as np
import pytest

from cnosdb_b200 import cabi, datagen
from cnosdb_b200.engine import CompactAggError, Engine, PushedAggregate, QueryOption, duration_in, state_at
from tests.state_periods_reference import handle_record, join, load_golden

pytestmark = pytest.mark.gpu
I64 = cabi.TSKV_PT_I64


@pytest.fixture(scope="module")
def eng():
    e = Engine(0)
    yield e
    e.close()


def one_series(eng, points, aggs=("state_agg",), **kw):
    """(duration map, periods) of the one cell of a series of points [(t, state)]."""
    b = datagen.ArenaBuilder()
    b.add_column_group(0, np.array([t for t, _ in points], np.int64), [(1, I64, np.array([s for _, s in points], np.int64), None, None)])
    a, d = b.finish()
    pages = eng.upload_pages(a, d)
    try:
        r = eng.scan_aggregate(pages, QueryOption([PushedAggregate(1, I64, list(aggs))], n_buckets=1, **kw))
        return r.state_maps(1)[0][0], (r.state_periods(1)[0][0] if "state_agg" in aggs else {})
    finally:
        pages.close()


def test_state_at_and_duration_in_slt(eng):
    g = load_golden()
    pts = sorted(((r["time"], r["code"]) for r in g["states"]["rows"]), key=lambda p: p[0])
    m, p = one_series(eng, pts)
    assert p == join(handle_record(pts))
    mc, pc = one_series(eng, pts, aggs=("compact_state_agg",))
    assert mc == m and pc == {}
    for e in g["state_at"]:
        if e["agg"] == "compact_state_agg":
            with pytest.raises(CompactAggError) as x:
                state_at(pc, e["ts"], mc)
            assert str(x.value) == e["error"], e["src"]
        else:
            assert state_at(p, e["ts"], m) == e["expected"], e["src"]
    for e in g["duration_in"]:
        end = None if e["interval"] is None else e["start"] + e["interval"]
        if e["agg"] == "compact_state_agg":
            with pytest.raises(CompactAggError) as x:
                duration_in(mc, e["code"], e["start"], end, pc)
            assert str(x.value) == e["error"], e["src"]
        else:
            assert duration_in(m, e["code"], e["start"], end, p) == e["expected"], e["src"]


def test_unit_fixture(eng):
    u = load_golden()["unit"]
    _, p = one_series(eng, [tuple(x) for x in u["points"]])
    assert p == join({s: [tuple(q) for q in ps] for s, ps in u["periods"]}), u["src"]
    assert p == {111: [(0, 3), (900, 1900)], 222: [(3, 100)], 333: [(100, 900)]}


def test_one_row_cell_is_the_compact_error(eng):
    m, p = one_series(eng, [(1_000, 3)])
    assert m == {3: 0} and p == {}
    with pytest.raises(CompactAggError):
        state_at(p, 1_000, m)
    with pytest.raises(CompactAggError):
        duration_in(m, 3, 0, 10_000, p)
    assert duration_in(m, 3) == 0  # (without a start time the map answers)
