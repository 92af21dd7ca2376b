"""tests/state_periods_reference.py against the reference's answers (state_at.slt, duration_in.slt with a start time, the
StatePeriods unit fixture), and the joined periods against the reference's periods: on random point lists, state_at and
duration_in give the same answers on both, for windows that cut a period, start before the first point or after the
last, have a zero interval or a NULL one; engine.state_at / engine.duration_in restate them on the joined periods."""
import numpy as np
import pytest

from cnosdb_b200 import engine
from tests import state_periods_reference as ref
from tests.state_agg_reference import fold

G = ref.load_golden()


def _states_points():
    return sorted(((r["time"], r["code"]) for r in G["states"]["rows"]), key=lambda p: p[0])


def test_unit_fixture_periods():
    raw = ref.handle_record([tuple(p) for p in G["unit"]["points"]])
    assert raw == {s: [tuple(p) for p in ps] for s, ps in G["unit"]["periods"]}
    # joined: 222's [3, 10) and [10, 100) touch
    assert ref.join(raw) == {111: [(0, 3), (900, 1900)], 222: [(3, 100)], 333: [(100, 900)]}


@pytest.mark.parametrize("case", range(len(G["state_at"])))
def test_state_at_golden(case):
    e = G["state_at"][case]
    pts = _states_points()
    raw, durs = ref.handle_record(pts), fold(pts)
    if e["agg"] == "compact_state_agg":  # the compact aggregate keeps no periods
        assert ref.is_compact({}, durs) and "error" in e
        with pytest.raises(engine.CompactAggError, match="doesn't support compact_agg"):
            engine.state_at({}, e["ts"], durs)
        return
    assert not ref.is_compact(raw, durs)
    assert ref.state_at(raw, e["ts"]) == e["expected"], e["src"]
    assert engine.state_at(ref.join(raw), e["ts"], durs) == e["expected"], e["src"]


@pytest.mark.parametrize("case", range(len(G["duration_in"])))
def test_duration_in_golden(case):
    e = G["duration_in"][case]
    pts = _states_points()
    raw, durs = ref.handle_record(pts), fold(pts)
    end = None if e["interval"] is None else e["start"] + e["interval"]
    if e["agg"] == "compact_state_agg":
        with pytest.raises(engine.CompactAggError) as x:
            engine.duration_in(durs, e["code"], e["start"], end, {})
        assert str(x.value) == e["error"]
        return
    assert ref.duration_in(raw, e["code"], e["start"], e["interval"]) == e["expected"], e["src"]
    assert engine.duration_in(durs, e["code"], e["start"], end, ref.join(raw)) == e["expected"], e["src"]


def test_one_row_cell_is_compact():
    pts = [(5, 1)]
    raw, durs = ref.handle_record(pts), fold(pts)
    assert raw == {} and durs == {1: 0} and ref.is_compact(raw, durs)
    with pytest.raises(engine.CompactAggError):
        engine.state_at(ref.join(raw), 5, durs)
    with pytest.raises(engine.CompactAggError):
        engine.duration_in(durs, 1, 0, None, ref.join(raw))
    # an empty cell is not compact: no state, 0
    assert engine.state_at({}, 5, {}) is None and engine.duration_in({}, 1, 0, 10, {}) == 0


def test_equal_times_cell():
    """Rows that all share one time: the reference has periods of length 0 (not compact: state_at NULL, duration_in 0);
    the joined periods are empty, so the scan's answer is the compact error."""
    pts = [(7, 1), (7, 2), (7, 1)]
    raw, durs = ref.handle_record(pts), fold(pts)
    assert raw == {1: [(7, 7)], 2: [(7, 7)]} and not ref.is_compact(raw, durs)
    assert ref.state_at(raw, 7) is None and ref.duration_in(raw, 1, 0, None) == 0
    assert ref.join(raw) == {} and ref.is_compact(ref.join(raw), durs)


@pytest.mark.parametrize("seed", range(40))
def test_joined_periods_answer_as_raw(seed):
    rng = np.random.default_rng(seed)
    pts = ref.random_points(rng, int(rng.integers(2, 60)))
    raw, durs = ref.handle_record(pts), fold(pts)
    joined = ref.join(raw)
    assert not ref.is_compact(raw, durs) and not ref.is_compact(joined, durs)
    # joined periods are maximal, positive and sorted; their lengths per state are the map's durations
    for s, ps in joined.items():
        assert all(a < b for a, b in ps) and all(ps[i][1] < ps[i + 1][0] for i in range(len(ps) - 1))
        assert sum(b - a for a, b in ps) == durs[s]
    t0, t1 = pts[0][0], pts[-1][0]
    cuts = sorted({t for t, _ in pts} | {t0 - 7, t1 + 7, (t0 + t1) // 2, t0 + 1, t1 - 1})
    starts = cuts + [t0 - 1000, t1 + 1000] + [int(x) for x in rng.integers(t0 - 10, t1 + 10, 10)]
    for start in starts:
        assert ref.state_at(raw, start) == ref.state_at(joined, start) == engine.state_at(joined, start, durs)
        for interval in (None, 0, 1, 3, int(rng.integers(1, t1 - t0 + 20)), t1 - t0 + 2000):
            for s in list(durs) + [99]:
                want = ref.duration_in(raw, s, start, interval)
                assert ref.duration_in(joined, s, start, interval) == want
                end = None if interval is None else start + interval
                assert engine.duration_in(durs, s, start, end, joined) == want
