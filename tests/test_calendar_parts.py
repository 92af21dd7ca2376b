"""calendar_parts (cnosdb_b200/engine.py): the labelled time buckets of GROUP BY date_part(unit, time) against the
reference's own date_part / extract expectations (tests/golden/date_part_slt.json) and against Python's datetime."""
import datetime
import json
import os

import numpy as np
import pytest

from cnosdb_b200.engine import PART_UNITS, calendar_parts

GOLDEN = os.path.join(os.path.dirname(__file__), "golden", "date_part_slt.json")
SCALE = {"s": 10**9, "ms": 10**6, "us": 10**3, "ns": 1}  # ns per unit
UNITS = tuple(PART_UNITS)
GOLD = json.load(open(GOLDEN))


def _ts(text, precision="ns"):
    """'YYYY-MM-DD[ T]HH:MM:SS[.fff]' (UTC) -> int timestamp in `precision` (floored)."""
    ns = int(np.datetime64(text.replace(" ", "T"), "ns").astype(np.int64))
    return ns // SCALE[precision]


def _part(edges, labels, values, t):
    """date_part of timestamp t by the labelled buckets: part_values[labels[bucket of t]]."""
    b = int(np.searchsorted(edges, t, side="right")) - 1
    assert 0 <= b < len(edges) - 1, (t, edges[0], edges[-1])
    return float(values[labels[b]])


def _check_shape(edges, labels, values, t_lo, t_hi):
    assert edges.dtype == np.int64 and labels.dtype == np.uint32 and values.dtype == np.float64
    assert edges.size >= 2 and labels.size == edges.size - 1
    assert (np.diff(edges) > 0).all()
    assert edges[0] <= t_lo and edges[-2] <= t_hi < edges[-1]
    assert int(labels.max()) < values.size
    assert (np.diff(values) > 0).all()  # one output bucket per value


def test_golden_covers_the_units():
    assert len(GOLD["files"]) == 2  # date_part.slt and extract.slt
    for f in GOLD["files"]:
        assert len(f["rows"]) == 5
        assert set(UNITS) <= {q["unit"] for q in f["queries"]}
    a, b = GOLD["files"]
    assert [r["time"] for r in a["rows"]] == [r["time"] for r in b["rows"]]
    assert [q["expected"] for q in a["queries"]] == [q["expected"] for q in b["queries"]]


@pytest.mark.parametrize("precision", ["s", "ms", "us", "ns"])
@pytest.mark.parametrize("unit", UNITS)
def test_slt_rows_get_the_expected_part(unit, precision):
    """Every slt timestamp's labelled bucket carries date_part's expected value: one table over all five rows (one per
    row and one over the two 2024 rows for hour and minute), from both files."""
    for f in GOLD["files"]:
        q = next(q for q in f["queries"] if q["unit"] == unit)
        times = [_ts(r["time"], precision) for r in f["rows"]]
        if unit in ("hour", "minute"):
            tables = [(calendar_parts(unit, t, t, precision), [i]) for i, t in enumerate(times)]
            tables.append((calendar_parts(unit, times[3], times[4], precision), [3, 4]))
        else:
            tables = [(calendar_parts(unit, min(times), max(times), precision), range(5))]
        for (edges, labels, values), rows in tables:
            _check_shape(edges, labels, values, min(times[i] for i in rows), max(times[i] for i in rows))
            for i in rows:
                assert _part(edges, labels, values, times[i]) == float(q["expected"][i]), (unit, f["rows"][i], q["src"])


def _expected(unit, dt):
    return {"year": dt.year, "quarter": (dt.month - 1) // 3 + 1, "month": dt.month, "week": dt.isocalendar()[1],
            "day": dt.day, "doy": dt.timetuple().tm_yday, "dow": (dt.weekday() + 1) % 7, "hour": dt.hour,
            "minute": dt.minute}[unit]


EPOCH = datetime.datetime(1970, 1, 1)


def _times(rng, n):
    """Random times from 1900 to 2100 (ns), plus leap days, ISO week 53 years and the days around New Year."""
    lo, hi = _ts("1900-01-01T00:00:00"), _ts("2100-12-31T23:59:59")
    ts = [int(x) for x in rng.integers(lo, hi, n)]
    for day in ("1904-02-29", "2000-02-29", "2024-02-29", "2020-12-31", "2021-01-03", "2026-12-31", "2027-01-03",
                "2015-12-31", "2016-01-03", "1969-12-31", "1970-01-01", "2009-12-31", "2010-01-03", "1900-12-31"):
        ts += [_ts(day + "T00:00:00"), _ts(day + "T23:59:59.999999999")]
    return ts


@pytest.mark.parametrize("unit", UNITS)
def test_random_times_against_datetime(unit):
    """Random times from 1900 to 2100 against datetime: isocalendar() (ISO week), weekday() (dow, 0 = Sunday),
    timetuple().tm_yday (doy). Tables over a few periods around each time, and one table over a whole ISO week 53
    year."""
    rng = np.random.default_rng(17 + len(unit))
    span = {"hour": 3 * 3600, "minute": 3 * 60}.get(unit, 40 * 86400) * 10**9
    for t in _times(rng, 60):
        edges, labels, values = calendar_parts(unit, t - span, t + span)
        _check_shape(edges, labels, values, t - span, t + span)
        dt = EPOCH + datetime.timedelta(microseconds=t // 1000)
        assert _part(edges, labels, values, t) == _expected(unit, dt), (unit, dt)
    # 2020 and 2026 have an ISO week 53 (they start on a Wednesday / Thursday); 2020 is a leap year. (Minutes: a year
    # of them is half a million edges; the random times above cover them.)
    for year in (2020, 2026) if unit != "minute" else ():
        lo, hi = _ts("%d-01-01T00:00:00" % year), _ts("%d-12-31T23:59:59" % year)
        edges, labels, values = calendar_parts(unit, lo, hi)
        for t in np.linspace(lo, hi, 97).astype(np.int64):
            dt = EPOCH + datetime.timedelta(microseconds=int(t) // 1000)
            assert _part(edges, labels, values, int(t)) == _expected(unit, dt), (unit, dt)


def test_week_53_and_day_366():
    edges, labels, values = calendar_parts("week", _ts("2020-12-28T00:00:00"), _ts("2021-01-04T00:00:00"))
    assert values[labels].tolist() == [53.0, 1.0]
    edges, labels, values = calendar_parts("doy", _ts("2024-12-31T00:00:00"), _ts("2024-12-31T00:00:00"))
    assert values[labels].tolist() == [366.0]


def test_cyclic_labels_fold_periods():
    """48 hours of hourly edges fold into 24 output buckets, each hour of the day twice; months into 12, days of the
    week into 7 - the output grid does not grow with the span."""
    lo = _ts("2024-01-01T00:00:00")
    edges, labels, values = calendar_parts("hour", lo, lo + 48 * 3600 * 10**9 - 1)
    assert edges.size - 1 == 48 and values.tolist() == list(range(24))
    assert np.bincount(labels, minlength=24).tolist() == [2] * 24
    edges, labels, values = calendar_parts("month", lo, _ts("2026-12-31T00:00:00"))
    assert labels.size == 36 and values.size == 12 and np.bincount(labels).tolist() == [3] * 12
    edges, labels, values = calendar_parts("dow", lo, lo + 13 * 86400 * 10**9)
    assert values.size == 7 and labels[:7].tolist() == [1, 2, 3, 4, 5, 6, 0]  # 2024-01-01 was a Monday
    edges, labels, values = calendar_parts("year", _ts("1968-05-01T00:00:00"), _ts("1971-02-01T00:00:00"))
    assert values.tolist() == [1968.0, 1969.0, 1970.0, 1971.0] and labels.tolist() == [0, 1, 2, 3]


@pytest.mark.parametrize("unit", ["second", "millisecond", "microsecond", "nanosecond", "epoch", "dom", "fortnight"])
def test_rejected_units(unit):
    with pytest.raises(ValueError):
        calendar_parts(unit, 0, 1)


def test_refusals():
    with pytest.raises(ValueError):
        calendar_parts("hour", 0, 1, precision="ps")
    with pytest.raises(ValueError):
        calendar_parts("day", 2, 1)
