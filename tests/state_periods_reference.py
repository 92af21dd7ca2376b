"""Exact per-cell state_agg(time, x) periods (TSKV_STATE_PERIODS) for arenas described by a `truth` dict, and restatements
of the reference's period functions (state_agg_data.rs, scalar_function/{state_at,duration_in}.rs).

`handle_record` restates StatePeriods::handle_record: for each pair of consecutive points (t, s), (t', s') in time order
it pushes the period [t, t') onto state s; the last point gets no period. `duration_in` and `state_at` restate
StateAggData::duration_in (with a start time) and ::state_at over such periods, and `is_compact` the rule of
StateAggData::try_from that makes both refuse an aggregate (no period, some duration entry).

The scan returns maximal periods instead (`join`): the periods of one state that touch end to end are joined, and
periods of length 0 are dropped. `exact_state_periods` selects each cell's points as tests/state_agg_reference.py does
and joins the reference's periods."""
import json
import os

import numpy as np

from tests.state_agg_reference import selected_points


def handle_record(points):
    """StatePeriods::handle_record over points [(t, state)] in time order -> {state: [(start, end)]}, each state's
    periods in the order they were pushed."""
    periods, last = {}, None
    for t, s in points:
        if last is not None:
            periods.setdefault(last[0], []).append((last[1], t))
        last = (s, t)
    return periods


def join(periods):
    """The maximal periods of {state: [(start, end)]}: sorted by start, length-0 periods dropped, and a period that
    starts where the previous one of its state ends joined to it. -> {state: [(start, end)]} without empty lists."""
    out = {}
    for s, ps in periods.items():
        cur = []
        for a, b in sorted(p for p in ps if p[1] > p[0]):
            if cur and cur[-1][1] == a:
                cur[-1] = (cur[-1][0], b)
            else:
                cur.append((a, b))
        if cur:
            out[s] = cur
    return out


def is_compact(periods, durations):
    """StateAggData::try_from: compact = periods.is_empty() && !durations.is_empty()."""
    return not periods and bool(durations)


def duration_in(periods, state, start, interval):
    """StateAggData::duration_in with a start time (interval None: a NULL interval): the lengths of the periods of
    `state` with end > start (and start < start + interval), each clipped to the window; 0 for an absent state."""
    total = 0
    if interval is not None:
        end = start + interval
        for a, b in periods.get(state, ()):
            if b > start and a < end:
                total += (end if b > end else b) - (start if a < start else a)
    else:
        for a, b in periods.get(state, ()):
            if b > start:
                total += b - (start if a < start else a)
    return total


def state_at(periods, ts):
    """StateAggData::state_at: the state of a period with start <= ts < end, None when there is none."""
    for s, ps in periods.items():
        if any(a <= ts < b for a, b in ps):
            return s
    return None


def exact_state_periods(truth, query, col, pt, n_cells, **kw):
    """[{state: [(start, end)]}] per cell: the joined periods of the cell's points (empty for a cell without rows)."""
    pts = selected_points(truth, query, col, pt, **kw)
    return [join(handle_record(pts.get(c, []))) for c in range(n_cells)]


def _ordered(d):
    """{state: periods} in the scan's order: the NULL state first, then the states by value."""
    return sorted(d.items(), key=lambda kv: (kv[0] is not None, kv[0] if kv[0] is not None else 0))


def check_state_periods(res, col, exact, what=""):
    """ScanResult `res`'s periods of state agg column `col` against exact_state_periods, exactly and in order."""
    got = [p for row in res.state_periods(col) for p in row]
    assert len(got) == len(exact), what
    bad = [(c, got[c], exact[c]) for c in range(len(exact)) if list(got[c].items()) != _ordered(exact[c])]
    assert not bad, (what, bad[:3])


def random_points(rng, n, n_states=4, max_step=5, null_frac=0.1):
    """n points [(t, state)] with strictly increasing times and runs of states (None: the NULL state)."""
    ts = np.cumsum(rng.integers(1, max_step + 1, n)) + int(rng.integers(-50, 50))
    out, s = [], 0
    for t in ts:
        if rng.random() < 0.4:
            s = None if rng.random() < null_frac else int(rng.integers(0, n_states))
        out.append((int(t), s))
    return out


# ---- the reference's answers (tests/golden/state_agg_periods_slt.json, written by make_state_agg_golden.py) ----
GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "state_agg_periods_slt.json")


def load_golden():
    with open(GOLDEN) as f:
        return json.load(f)
