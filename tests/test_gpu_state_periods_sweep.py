"""state_agg periods over every fused-scan bin and over seeded random query combinations (gauges, modes, increases, pairs,
tombstones, chunk files, predicates, host-resident and verify-on-read page sets): every output, every duration map and
the counters equal those of the same scan with the operands unflagged (compact_state_agg), and every cell's periods
equal tests/state_periods_reference.py's joined periods.

1. test_every_bin: sweep_reference.bin_arena's arena of every bin, grouped by series on tumbling and edge grids, with a
   state_agg of every integer column. Every bin but the Gorilla ones (f64 pages only) must run.
2. test_random_combinations: sweep_reference.random_operand_case cases grouped by series, with 1-3 state aggs (each a
   state_agg, a compact_state_agg or both) and a gauge, a mode and an increase, until N_CASES cases ran."""
import copy

import numpy as np
import pytest

from cnosdb_b200 import cabi
from cnosdb_b200.engine import Engine, PushedAggregate, TskvError
from tests import sweep_reference as sw
from tests.state_agg_reference import check_state_maps, exact_state_maps
from tests.state_periods_reference import check_state_periods, exact_state_periods
from tests.test_gpu_kernel_sweep import scan_kwargs, set_env

pytestmark = pytest.mark.gpu

BASE_SEED = 20261020
N_CASES = 80
INTS = (cabi.TSKV_PT_I64, cabi.TSKV_PT_U64)
COUNTERS = ("page_read_count", "page_read_bytes", "points_decoded", "rows_in_range", "pruned_page_count")


@pytest.fixture(scope="module")
def engine():
    e = Engine(0)
    yield e
    e.close()


def unflagged(q):
    """q with every state_agg asked as compact_state_agg: the same operands without TSKV_STATE_PERIODS."""
    q0 = copy.copy(q)
    q0.columns, q0._keep = [], None
    for c in q.columns:
        if getattr(c, "state_agg", False):
            c = copy.copy(c)
            c.state_agg, c.compact_state_agg = False, True
        q0.columns.append(c)
    return q0


def compare(engine, pages, q, truth, extra, what, tombstones=None, files=None):
    kw = scan_kwargs(extra)
    got = engine.scan_aggregate(pages, q, **kw)
    c1 = engine.counters()
    base = engine.scan_aggregate(pages, unflagged(q), **kw)
    c0 = engine.counters()
    assert got.names == base.names, what
    np.testing.assert_array_equal(got.validity, base.validity, err_msg=what)
    for j, name in enumerate(base.names):  # (f64 sums may differ in their last bits from run to run)
        ok = base.validity[j]
        x, y = got.values[j][ok], base.values[j][ok]
        pt = got.phys.get(name[0])
        if name[1] in ("mean", "m2", "c", "m2x", "m2y") or (pt == cabi.TSKV_PT_F64 and name[1] in ("sum", "increase")):
            np.testing.assert_allclose(x.view(np.float64), y.view(np.float64), rtol=1e-9, atol=1e-300, err_msg="%s %s" % (what, name))
        else:
            np.testing.assert_array_equal(x, y, err_msg="%s %s" % (what, name))
    for k in COUNTERS:
        assert c1[k] == c0[k], (what, k)
    assert set(got.state_csr) == set(base.state_csr), what
    for c in got.state_csr:
        assert all(x.tobytes() == y.tobytes() for x, y in zip(got.state_csr[c], base.state_csr[c])), what
    n_cells = got.n_groups * got.n_buckets
    kw_ref = dict(tombstones=tombstones, files=files, group_ids=extra.get("group_ids"), edges=extra.get("edges"))
    for (cid, pt), periods in zip(q.state_aggs(), q.state_periods()):
        check_state_maps(got, cid, exact_state_maps(truth, q, cid, pt, n_cells, **kw_ref), "%s map of %d" % (what, cid))
        if periods:
            exact = exact_state_periods(truth, q, cid, pt, n_cells, **kw_ref)
            check_state_periods(got, cid, exact, "%s periods of %d" % (what, cid))
    assert set(got.period_csr) == {cid for (cid, _), p in zip(q.state_aggs(), q.state_periods()) if p}, what
    again = engine.scan_aggregate(pages, q, **kw)  # the periods, byte for byte
    for c in got.period_csr:
        assert all(x.tobytes() == y.tobytes() for x, y in zip(again.period_csr[c], got.period_csr[c])), what


def test_every_bin(engine, monkeypatch):
    set_env(monkeypatch, {"TSKV_PARTS": None, "TSKV_SMEM_TABLE_KB": None})
    ran, expect = set(), set()
    for b in range(sw.N_BINS):
        tk, vk = divmod(sw.serial_bin(b), sw.N_VK)
        s8b = vk == sw.VK_S8B and tk != sw.TK_GEN
        for narrow in ((sw.NARROW_NONE, sw.NARROW_SOME, sw.NARROW_ALL) if s8b else (sw.NARROW_NONE,)):
            if vk != sw.VK_GOR:  # (Gorilla pages hold f64 values only: no state agg operand lands in those bins)
                expect |= {(b, narrow, False), (b, narrow, True)}
            arena, descs, truth = sw.bin_arena(b, narrow)
            ints = [c for c in sw.columns_of(truth) if sw.COLUMNS[c] in INTS]
            if not ints:
                continue
            for edges in (False, True):
                q, extra = sw.targeted_query(truth, (sw.SCAN, tk, vk, False, narrow, edges), seed=b)
                q.group_by_series = True
                extra.pop("group_ids", None)
                extra.pop("n_groups", None)
                q.columns += [PushedAggregate(c, sw.COLUMNS[c], ["state_agg"]) for c in ints]
                what = "state periods in bin %d narrow %d edges %s" % (b, narrow, edges)
                pages = engine.upload_pages(arena, descs)
                try:
                    compare(engine, pages, q, truth, extra, what)
                    ran.add((b, narrow, edges))
                finally:
                    pages.close()
    assert ran == expect, (sorted(expect - ran), sorted(ran - expect))


def add_operands(q, truth, rng):
    """1-3 state aggs of the arena's integer columns (state_agg, compact_state_agg or both), and maybe a gauge, a mode
    and an increase. False when the arena has no integer column."""
    ints = [c for c in sw.columns_of(truth) if sw.COLUMNS[c] in INTS]
    num = [c for c in sw.columns_of(truth) if sw.COLUMNS[c] != sw.BOOL]
    if not ints:
        return False
    kinds = (["state_agg"], ["state_agg"], ["compact_state_agg"], ["state_agg", "compact_state_agg"])
    for _ in range(int(rng.integers(1, 4))):
        c = int(rng.choice(ints))
        q.columns.append(PushedAggregate(c, sw.COLUMNS[c], kinds[int(rng.integers(0, len(kinds)))]))
    for kind in ("gauge_agg", "mode", "increase"):
        if rng.random() < 0.5:
            c = int(rng.choice(num))
            q.columns.append(PushedAggregate(c, sw.COLUMNS[c], [kind]))
    return True


def test_random_combinations(engine, monkeypatch):
    ran, i, outcomes = 0, 0, {}
    while ran < N_CASES:
        assert i < 6 * N_CASES, "too few random cases take state aggs: %d of %d" % (ran, i)
        case = sw.random_operand_case(i, BASE_SEED)
        i += 1
        base = sw.case_expected(case)
        if isinstance(base, (int, str)) or "slide" in case.extra or "labels" in case.extra or \
                any(c.median for c in case.query.columns) and case.query.n_buckets * 2000 > (1 << 22) or \
                not add_operands(case.query, case.truth, np.random.default_rng([BASE_SEED, i, 7])):
            outcomes["skipped"] = outcomes.get("skipped", 0) + 1
            continue
        q = case.query
        if not any(q.state_periods()):
            outcomes["skipped"] = outcomes.get("skipped", 0) + 1
            continue
        q.group_by_series = "group_ids" not in case.extra
        what = case.describe()
        set_env(monkeypatch, case.env)
        pages = engine.upload_pages(case.arena, case.descs, host_resident=case.host_resident, verify_on_read=case.verify_on_read)
        try:
            if case.tombstones is not None:
                pages.set_tombstones(case.tombstones)
            if case.files is not None:
                pages.set_chunk_files(case.files)
            try:
                compare(engine, pages, q, case.truth, case.extra, what, tombstones=case.tombstones, files=case.files)
            except TskvError as e:
                # a tag group of two series, or a column group without the operand: refused as documented
                assert e.status == cabi.TSKV_ERR_UNSUPPORTED, (what, e)
                outcomes["refused"] = outcomes.get("refused", 0) + 1
                continue
        finally:
            pages.close()
        ran += 1
        shape = case.desc.get("grouping", "?")
        outcomes[shape] = outcomes.get(shape, 0) + 1
    print("\nrandom state period combinations: %d cases over %d drawn; %s" % (ran, i, outcomes))
