"""FIRST / LAST runs and tombstone range edges through the fused scan against the exact reference (tests/helpers.py),
bit for bit, on the arenas of tests/exact_arenas.py: RLE, jittered simple8b and raw time pages; narrow / wide simple8b,
Gorilla, raw and boolean value pages; NULLs at runs' first / last rows, equal times across slots, predicates that drop
a run's first row, several column groups per series, the 62-bit key budget at 61 / 62 / 63 bits; tombstone edges on,
one before and one after rows at bucket edges, restart-point cuts, page ends and the i64 limits. Every query runs with
pages whole and cut into 3 parts, by bucket, by series, by tags and unbucketed; one per arena as a two-shard exchange."""
import functools

import numpy as np
import pytest

from cnosdb_b200 import cabi
from cnosdb_b200.engine import TskvError
from tests import exact_arenas as ea
from tests.helpers import assert_matches_exact, exact_aggregate
from tests.ranks import sharded_scans, with_series

pytestmark = pytest.mark.gpu

ENVS = ("1", "3")  # TSKV_PARTS


@functools.lru_cache(maxsize=None)
def fl_arena(kind):
    return ea.first_last_arena(kind)


@functools.lru_cache(maxsize=None)
def tomb_arena(step, kind):
    arena, descs, truth = ea.tombstone_arena(step, kind)
    return arena, descs, truth, ea.tombstone_list(truth, step)


def _scan(engine, pages, q, extra):
    return engine.scan_aggregate(pages, q, group_ids=extra.get("group_ids"), n_groups=extra.get("n_groups"))


@pytest.mark.parametrize("kind", ea.FL_KINDS)
def test_first_last_runs(engine, kind, monkeypatch):
    arena, descs, truth = fl_arena(kind)
    pages = engine.upload_pages(arena, descs)
    for name, q, extra in ea.first_last_queries(truth):
        exp = ea.expected(truth, q, extra)
        for parts in ENVS:
            monkeypatch.setenv("TSKV_PARTS", parts)
            assert_matches_exact(_scan(engine, pages, q, extra), exp, what="%s %s parts=%s" % (kind, name, parts))
    pages.close()
    monkeypatch.setenv("TSKV_PARTS", ENVS[0])
    ids = np.arange(ea.FL_SERIES, dtype=np.uint32)
    for name, q, _ in ea.first_last_queries(truth)[:5]:
        if q.width == 0:
            continue
        q = q if q.series_ids is not None else with_series(q, ids)
        exp = exact_aggregate(truth, q)
        for got in sharded_scans(engine, arena, descs, q, (ids[ids % 2 == 0], ids[ids % 2 == 1])):
            assert_matches_exact(got, exp, what="%s %s 2-shard exchange" % (kind, name), int_mean=False)


@pytest.mark.parametrize("width,bits", ea.BUDGET_WIDTHS)
def test_first_last_key_budget(engine, width, bits):
    cases = [(ea.key_budget_arena(width), ea.key_budget_queries(width)[0][1], bits)]
    if bits == 62:
        cases += [(ea.key_budget_arena(None, 2**60 - 1), ea.key_budget_queries(None, True)[0][1], 62),
                  (ea.key_budget_arena(None, 2**60), ea.key_budget_queries(None, True)[0][1], 63)]
    for (arena, descs, truth), q, b in cases:
        pages = engine.upload_pages(arena, descs)
        if b > 62:
            with pytest.raises(TskvError) as e:
                engine.scan_aggregate(pages, q)
            assert e.value.status == cabi.TSKV_ERR_UNSUPPORTED
        else:
            assert_matches_exact(engine.scan_aggregate(pages, q), exact_aggregate(truth, q), what="width %s" % width)
        pages.close()


@pytest.mark.parametrize("step,kind", ea.TB_CASES)
def test_tombstone_edges(engine, step, kind, monkeypatch):
    arena, descs, truth, tombs = tomb_arena(step, kind)
    pages = engine.upload_pages(arena, descs)
    pages.set_tombstones(tombs)
    host = engine.upload_pages(arena, descs, host_resident=True)
    host.set_tombstones(tombs)
    for name, q, extra in ea.tombstone_queries(truth, step):
        exp = ea.expected(truth, q, extra, tombstones=tombs)
        for parts in ENVS:
            monkeypatch.setenv("TSKV_PARTS", parts)
            assert_matches_exact(_scan(engine, pages, q, extra), exp, what="step %d %s %s parts=%s" % (step, kind, name, parts))
        monkeypatch.setenv("TSKV_PARTS", ENVS[0])
        assert_matches_exact(_scan(engine, host, q, extra), exp, what="step %d %s %s host-resident" % (step, kind, name))
    host.close()
    pages.close()
    q = ea.tombstone_queries(truth, step)[0][1]
    ids = q.series_ids
    exp = exact_aggregate(truth, q, tombstones=tombs)
    for got in sharded_scans(engine, arena, descs, q, (ids[:5], ids[5:]), tombstones=tombs):
        assert_matches_exact(got, exp, what="step %d %s 2-shard exchange" % (step, kind), int_mean=False)
