"""The reference's gauge_agg / delta / rate / time_delta / idelta_* / first_* / last_* answers (tests/golden/gauge_slt.json)
through the scan: each answer's table written as one column group per series (its tag set), every numeric field a
column of its type (func_tb2.f0 BIGINT UNSIGNED included), GROUP BY t0 as a tag-group map and GROUP BY
date_trunc('day', time) as one-day buckets; the nine outputs read through ScanResult.gauge and the accessors derived by
engine.gauge_stat. The tables hold no timestamp tie within a group. The operand types the reference refuses at planning
(Boolean, Utf8, Timestamp) are refused before any launch or have no page type."""
import numpy as np
import pytest

from cnosdb_b200 import cabi, datagen
from cnosdb_b200.engine import GAUGE_OUTS, Engine, PushedAggregate, QueryOption, TskvError
from tests.gauge_reference import DAY, golden_cases, golden_refused

pytestmark = pytest.mark.gpu

CASES = golden_cases()
DT = {cabi.TSKV_PT_I64: np.int64, cabi.TSKV_PT_U64: np.uint64, cabi.TSKV_PT_F64: np.float64}


@pytest.fixture(scope="module")
def eng():
    e = Engine(0)
    yield e
    e.close()


def case_arena(case):
    """(arena, descs, field -> column id) of a GaugeGolden: one column group per series in series() order."""
    ids = {f: k + 1 for k, f in enumerate(sorted(case.types))}
    b = datagen.ArenaBuilder()
    for sid, tags in enumerate(case.series()):
        rows = sorted((t, v) for t, tg, v in case.rows if tg == tags)
        ts = np.array([t for t, _ in rows], dtype=np.int64)
        fields = []
        for f, pt in case.types.items():
            vals = np.array([0 if v.get(f) is None else v[f] for _, v in rows], dtype=DT[pt])
            valid = np.array([v.get(f) is not None for _, v in rows], dtype=bool)
            fields.append((ids[f], pt, vals, valid, None))
        b.add_column_group(sid, ts, fields)
    arena, descs = b.finish()
    return arena, descs, ids


@pytest.mark.parametrize("k", range(len(CASES)))
def test_golden_answers(eng, k):
    case = CASES[k]
    arena, descs, ids = case_arena(case)
    fields = sorted({it[1] for it in case.items if it})
    pages = eng.upload_pages(arena, descs)
    try:
        series = case.series()
        q = QueryOption([PushedAggregate(ids[f], case.types[f], ["gauge_agg"]) for f in fields],
                        series_ids=np.arange(len(series), dtype=np.uint32), n_buckets=1)
        kw = {}
        if case.group == "t0":
            keys = case.groups()
            t0 = case.tags.index("t0")
            kw = dict(group_ids=np.array([keys.index(s[t0]) for s in series], dtype=np.uint32), n_groups=len(keys))
        elif case.group == "day":
            days = case.groups()
            q.width, q.first_bucket_start, q.n_buckets = DAY, days[0] * DAY, days[-1] - days[0] + 1
        res = eng.scan_aggregate(pages, q, **kw)

        def outputs(field):
            cols = [res.gauge(ids[field], g) for g in GAUGE_OUTS]
            vals = [c[0].ravel() for c in cols]
            if case.group == "day":
                keep = [d - case.groups()[0] for d in case.groups()]
                vals = [v[keep] for v in vals]
            return [tuple(int(v[i]) if j == 0 or j % 2 else float(v[i]) for j, v in enumerate(vals)) for i in range(len(vals[0]))]
        case.check(outputs)
    finally:
        pages.close()


def test_refused_types(eng):
    assert golden_refused() == ["Boolean", "Timestamp", "Utf8"]
    arena, descs, _ = case_arena(CASES[0])
    pages = eng.upload_pages(arena, descs)
    try:
        for pt in (cabi.TSKV_PT_TIME, cabi.TSKV_PT_BOOL):
            with pytest.raises(TskvError) as e:
                eng.scan_aggregate(pages, QueryOption([PushedAggregate(1, pt, ["gauge_agg"])], n_buckets=1))
            assert e.value.status == cabi.TSKV_ERR_INVALID_ARG
    finally:
        pages.close()
