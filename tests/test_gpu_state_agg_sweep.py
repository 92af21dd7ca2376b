"""compact_state_agg over every fused-scan bin and over seeded random query combinations (gauges, modes, medians,
increases, pairs, tombstones, chunk files, predicates, host-resident and verify-on-read page sets): every other output
equals that of the same scan without state aggs, and every map equals tests/state_agg_reference.py's.

1. test_every_bin: sweep_reference.bin_arena's arena of every bin (time class x value encoding; the simple8b bins with
   wide, mixed and narrow pages), grouped by series on tumbling and edge grids, with a state agg of every integer column.
   Every bin but the Gorilla ones (f64 pages only) must run.
2. test_random_combinations: sweep_reference.random_operand_case cases grouped by series, with 1-3 state aggs and a
   gauge, a mode and an increase added from a stream of their own, until N_CASES cases ran."""
import copy

import numpy as np
import pytest

from cnosdb_b200 import cabi
from cnosdb_b200.engine import Engine, PushedAggregate, TskvError
from tests import sweep_reference as sw
from tests.state_agg_reference import check_state_maps, exact_state_maps
from tests.test_gpu_kernel_sweep import scan_kwargs, set_env

pytestmark = pytest.mark.gpu

BASE_SEED = 20261019
N_CASES = 100
INTS = (cabi.TSKV_PT_I64, cabi.TSKV_PT_U64)


@pytest.fixture(scope="module")
def engine():
    e = Engine(0)
    yield e
    e.close()


def without_states(q):
    q0 = copy.copy(q)
    q0.columns, q0._keep = [c for c in q.columns if not c.compact_state_agg], None
    return q0


def compare(engine, pages, q, truth, extra, what, tombstones=None, files=None):
    """Runs q and q without its state aggs: the shared outputs agree, the maps equal the reference's."""
    kw = scan_kwargs(extra)
    got = engine.scan_aggregate(pages, q, **kw)
    base = engine.scan_aggregate(pages, without_states(q), **kw)
    n0 = len(base.names)
    assert got.names[:n0] == base.names, what
    for j, name in enumerate(base.names):
        np.testing.assert_array_equal(got.validity[j], base.validity[j], err_msg="%s %s" % (what, name))
        ok = base.validity[j]
        x, y = got.values[j][ok], base.values[j][ok]
        pt = got.phys.get(name[0])
        if name[1] in ("mean", "m2", "c", "m2x", "m2y") or (pt == cabi.TSKV_PT_F64 and name[1] in ("sum", "increase")):
            np.testing.assert_allclose(x.view(np.float64), y.view(np.float64), rtol=1e-9, atol=1e-300, err_msg="%s %s" % (what, name))
        else:
            np.testing.assert_array_equal(x, y, err_msg="%s %s" % (what, name))
    n_cells = got.n_groups * got.n_buckets
    for cid, pt in q.state_aggs():
        exact = exact_state_maps(truth, q, cid, pt, n_cells, tombstones=tombstones, files=files,
                                 group_ids=extra.get("group_ids"), edges=extra.get("edges"))
        check_state_maps(got, cid, exact, "%s state agg of %d" % (what, cid))
    again = engine.scan_aggregate(pages, q, **kw)  # the maps and their entry counts, byte for byte
    for j, name in enumerate(got.names[n0:], n0):
        np.testing.assert_array_equal(again.values[j], got.values[j], err_msg="%s %s" % (what, name))
    assert all(again.state_csr[c][k].tobytes() == got.state_csr[c][k].tobytes() for c in got.state_csr for k in range(4)), what


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
                q.columns += [PushedAggregate(c, sw.COLUMNS[c], ["compact_state_agg"]) for c in ints]
                what = "state aggs in bin %d narrow %d edges %s" % (b, narrow, edges)
                pages = engine.upload_pages(arena, descs)
                try:
                    compare(engine, pages, q, truth, extra, what)
                    ran.add((b, narrow, edges))
                finally:
                    pages.close()
    assert ran == expect, (sorted(expect - ran), sorted(ran - expect))


def add_operands(q, truth, rng):
    """1-3 state aggs of the arena's integer columns, and maybe a gauge, a mode and an increase. False when the arena has
    no integer column."""
    ints = [c for c in sw.columns_of(truth) if sw.COLUMNS[c] in INTS]
    num = [c for c in sw.columns_of(truth) if sw.COLUMNS[c] != sw.BOOL]
    if not ints:
        return False
    for _ in range(int(rng.integers(1, 4))):
        c = int(rng.choice(ints))
        q.columns.append(PushedAggregate(c, sw.COLUMNS[c], ["compact_state_agg"]))
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
    print("\nrandom state agg combinations: %d cases over %d drawn; %s" % (ran, i, outcomes))
