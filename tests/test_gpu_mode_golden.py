"""The reference's mode.slt and approx_distinct.slt answers (tests/golden/mode_slt.json) through the scan: each answer's
table written as one column group per series (its tag set), the WHERE x IN (v) as a predicate x == v, GROUP BY t0 as a
tag-group map; and the operand types mode.slt answers but the scan refuses (TIME, BOOLEAN; string and geometry columns
have no page type here)."""
import numpy as np
import pytest

from cnosdb_b200 import cabi, datagen
from cnosdb_b200.engine import Engine, PushedAggregate, QueryOption, TskvError
from tests.mode_reference import golden_cases, golden_refused

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def eng():
    e = Engine(0)
    yield e
    e.close()


def case_arena(case):
    """(arena, descs, series tags in slot order) of a GoldenCase: column 1 holds the value, NULL where it is None."""
    series = sorted({tags for _, tags, _ in case.rows})
    b = datagen.ArenaBuilder()
    dt = {cabi.TSKV_PT_I64: np.int64, cabi.TSKV_PT_U64: np.uint64, cabi.TSKV_PT_F64: np.float64}[case.pt]
    for sid, tags in enumerate(series):
        rows = sorted((t, v) for t, tg, v in case.rows if tg == tags)
        ts = np.array([t for t, _ in rows], dtype=np.int64)
        vals = np.array([0 if v is None else v for _, v in rows], dtype=dt)
        valid = np.array([v is not None for _, v in rows], dtype=bool)
        b.add_column_group(sid, ts, [(1, case.pt, vals, valid, None)])
    arena, descs = b.finish()
    return arena, descs, series


@pytest.mark.parametrize("k", range(8))
def test_golden_answers(eng, k):
    case = golden_cases()[k]
    arena, descs, series = case_arena(case)
    pages = eng.upload_pages(arena, descs)
    try:
        agg = "mode" if case.kind == "mode" else "count_distinct"
        preds = [(1, case.pt, "==", case.pred)] if case.pred is not None else []
        q = QueryOption([PushedAggregate(1, case.pt, [agg])], series_ids=np.arange(len(series), dtype=np.uint32),
                        n_buckets=1, predicates=preds)
        kw = {}
        if case.group_tag is not None:
            keys = sorted({tags[case.group_tag] for tags in series})
            kw = dict(group_ids=np.array([keys.index(t[case.group_tag]) for t in series], dtype=np.uint32), n_groups=len(keys))
        res = eng.scan_aggregate(pages, q, **kw)
        v, ok = res.column(1, agg)
        assert ok.all(), case.what
        assert v.ravel().tolist() == case.expected, (case.what, v.ravel().tolist(), case.expected)
    finally:
        pages.close()


def test_refused_types(eng):
    """TIME and BOOLEAN operands are refused before any launch; string and geometry columns have no page type."""
    case = golden_cases()[0]
    arena, descs, _ = case_arena(case)
    types = {t for _, t, _ in golden_refused()}
    assert types == {"TIME", "BOOLEAN", "STRING", "GEOMETRY"}
    pages = eng.upload_pages(arena, descs)
    try:
        for pt in (cabi.TSKV_PT_TIME, cabi.TSKV_PT_BOOL):
            for agg in ("mode", "count_distinct"):
                with pytest.raises(TskvError) as e:
                    eng.scan_aggregate(pages, QueryOption([PushedAggregate(1, pt, [agg])], n_buckets=1))
                assert e.value.status == cabi.TSKV_ERR_INVALID_ARG
    finally:
        pages.close()
