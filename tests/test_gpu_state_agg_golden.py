"""The reference's compact_state_agg answers (tests/golden/compact_state_agg_slt.json) through the scan: duration_in.slt's
states table, its string states coded to i64, and the DurationStates unit fixture of state_agg_data.rs."""
import numpy as np
import pytest

from cnosdb_b200 import cabi, datagen
from cnosdb_b200.engine import Engine, PushedAggregate, QueryOption, duration_in
from tests.state_agg_reference import load_golden

pytestmark = pytest.mark.gpu
I64 = cabi.TSKV_PT_I64


@pytest.fixture(scope="module")
def eng():
    e = Engine(0)
    yield e
    e.close()


def one_series_map(eng, points, **kw):
    b = datagen.ArenaBuilder()
    ts = np.array([t for t, _ in points], dtype=np.int64)
    v = np.array([s for _, s in points], dtype=np.int64)
    b.add_column_group(0, ts, [(1, I64, v, None, None)])
    a, d = b.finish()
    pages = eng.upload_pages(a, d)
    try:
        r = eng.scan_aggregate(pages, QueryOption([PushedAggregate(1, I64, ["compact_state_agg"])], n_buckets=1, **kw))
        return r.state_maps(1)[0][0]
    finally:
        pages.close()


def test_duration_in_slt(eng):
    g = load_golden()
    m = one_series_map(eng, [(r["time"], r["code"]) for r in g["states"]["rows"]])
    for a in g["answers"]:
        assert duration_in(m, a["code"]) == a["expected"], a["src"]
    assert len(m) == len(g["states"]["codes"])


def test_unit_fixture(eng):
    u = load_golden()["unit"]
    m = one_series_map(eng, [(t, s) for t, s in u["points"]])
    assert m == {s: d for s, d in u["durations"]}, u["src"]
