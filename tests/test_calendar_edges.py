"""calendar_edges (cnosdb_b200/engine.py): the time-bucket edges of GROUP BY date_trunc(unit, time) against the
reference's own date_trunc expectations (tests/golden/date_trunc_slt.json) and against hand-checked calendar facts."""
import json
import os

import numpy as np
import pytest

from cnosdb_b200.engine import CALENDAR_UNITS, calendar_edges

GOLDEN = os.path.join(os.path.dirname(__file__), "golden", "date_trunc_slt.json")
SCALE = {"ms": 10**6, "us": 10**3, "ns": 1}  # ns per unit


def _ts(text, precision="ns"):
    """'YYYY-MM-DD[ T]HH:MM:SS[.fff]' (UTC) -> int timestamp in `precision`."""
    ns = int(np.datetime64(text.replace(" ", "T"), "ns").astype(np.int64))
    assert ns % SCALE[precision] == 0
    return ns // SCALE[precision]


def _bucket_start(edges, t):
    b = int(np.searchsorted(edges, t, side="right")) - 1
    assert 0 <= b < len(edges) - 1, (t, edges[0], edges[-1])
    return int(edges[b])


def _check_edges(edges, t_lo, t_hi):
    e = np.asarray(edges)
    assert e.dtype == np.int64 and e.size >= 2
    assert (np.diff(e) > 0).all()
    assert e[0] <= t_lo and e[-1] > t_hi and e[-2] <= t_hi


GOLD = json.load(open(GOLDEN))


def test_golden_covers_every_unit():
    assert [q["unit"] for q in GOLD["queries"]] == list(CALENDAR_UNITS)
    assert len(GOLD["rows"]) == 5


@pytest.mark.parametrize("precision", ["ms", "us", "ns"])
@pytest.mark.parametrize("unit", CALENDAR_UNITS)
def test_slt_rows_land_in_the_expected_bucket(unit, precision):
    """Every slt timestamp lies in the bucket whose start is date_trunc's expected value (one edge table over all five
    rows, and one per row)."""
    q = next(q for q in GOLD["queries"] if q["unit"] == unit)
    times = [_ts(r["time"], precision) for r in GOLD["rows"]]
    if unit in ("hour", "minute", "second"):
        # one table over 64 years of seconds is large: one table per row and one over the two 2024 rows
        tables = [(calendar_edges(unit, t, t, precision), [i]) for i, t in enumerate(times)]
        tables.append((calendar_edges(unit, times[3], times[4], precision), [3, 4]))
    else:
        tables = [(calendar_edges(unit, min(times), max(times), precision), range(5))]
    for edges, rows in tables:
        _check_edges(edges, min(times[i] for i in rows), max(times[i] for i in rows))
        for i in rows:
            assert _bucket_start(edges, times[i]) == _ts(q["expected"][i], precision), (unit, GOLD["rows"][i])


@pytest.mark.parametrize("precision", ["ms", "us", "ns"])
def test_february_leap_years(precision):
    """2000 is a leap year (divisible by 400), 1900 is not (divisible by 100): February has 29 / 28 days."""
    day = 86400 * 10**9 // SCALE[precision]
    for year, days in ((2000, 29), (1900, 28), (2024, 29), (2023, 28)):
        lo = _ts("%d-02-10T00:00:00" % year, precision)
        e = calendar_edges("month", lo, lo, precision)
        assert list(e) == [_ts("%d-02-01T00:00:00" % year, precision), _ts("%d-03-01T00:00:00" % year, precision)]
        assert (e[1] - e[0]) == days * day
    y = calendar_edges("year", _ts("1900-06-01T00:00:00", precision), _ts("1901-01-01T00:00:00", precision), precision)
    assert (y[1] - y[0]) == 365 * day


@pytest.mark.parametrize("precision", ["ms", "us", "ns"])
def test_before_1970_floors(precision):
    """Times before the epoch go to the unit start at or before them (floor), never towards zero."""
    one = SCALE["ms"] // SCALE[precision]  # 1 ms in `precision`
    t = -one  # 1969-12-31T23:59:59.999
    assert _bucket_start(calendar_edges("year", t, t, precision), t) == _ts("1969-01-01T00:00:00", precision)
    assert _bucket_start(calendar_edges("quarter", t, t, precision), t) == _ts("1969-10-01T00:00:00", precision)
    assert _bucket_start(calendar_edges("month", t, t, precision), t) == _ts("1969-12-01T00:00:00", precision)
    assert _bucket_start(calendar_edges("week", t, t, precision), t) == _ts("1969-12-29T00:00:00", precision)  # Monday
    assert _bucket_start(calendar_edges("day", t, t, precision), t) == _ts("1969-12-31T00:00:00", precision)
    assert _bucket_start(calendar_edges("second", t, t, precision), t) == _ts("1969-12-31T23:59:59", precision)
    # exactly on a unit start: that unit, and the next edge is the following unit
    t0 = _ts("1960-03-01T00:00:00", precision)
    e = calendar_edges("month", t0, t0, precision)
    assert list(e) == [t0, _ts("1960-04-01T00:00:00", precision)]


def test_weeks_start_on_monday():
    """(numpy's datetime64[W] weeks start on Thursday 1970-01-01: not what date_trunc does)"""
    for day in ("1960-12-26", "1999-12-27", "2024-08-05", "1970-01-05", "1969-12-29"):
        t = _ts(day + "T12:00:00")
        assert _bucket_start(calendar_edges("week", t, t), t) == _ts(day + "T00:00:00")
        assert np.datetime64(day).astype("datetime64[D]").item().weekday() == 0


@pytest.mark.parametrize("unit", CALENDAR_UNITS)
def test_span_cover_and_count(unit):
    """Multi-year spans: strictly increasing, covering [t_lo, t_hi], each bucket one unit long."""
    lo, hi = _ts("1968-11-15T13:14:15"), _ts("1971-02-03T04:05:06")
    if unit in ("minute", "second"):
        hi = lo + 3 * 86400 * 10**9
    e = calendar_edges(unit, lo, hi)
    _check_edges(e, lo, hi)
    n = {"year": 4, "quarter": 10, "month": 28}.get(unit)
    if n is not None:
        assert e.size - 1 == n
    if unit == "month":
        starts = [np.datetime64(int(x), "ns").astype("datetime64[D]").item() for x in e]
        assert all(d.day == 1 for d in starts)


def test_refusals():
    with pytest.raises(ValueError):
        calendar_edges("fortnight", 0, 1)
    with pytest.raises(ValueError):
        calendar_edges("day", 0, 1, precision="ps")
    with pytest.raises(ValueError):
        calendar_edges("day", 2, 1)
