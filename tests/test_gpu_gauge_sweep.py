"""gauge_agg(time, x) over every fused-scan bin and over random query combinations, against tests/gauge_reference.py bit
for bit:

1. test_every_bin: sweep_reference.bin_arena's arena of every bin (time class x value encoding; the simple8b bins with
   wide, mixed and narrow pages, the generic bin's short, run-length and all-NULL pages), tumbling and edge grids, with a
   gauge of every numeric column and a second gauge of the first.
2. test_random_combinations: seeded sweep_reference.random_operand_case cases (pairs, medians, tombstones, chunk files,
   predicates, host-resident and verify-on-read page sets, every grouping but sliding windows), some with modes and
   distincts added as tests/test_gpu_mode_sweep.py adds them, with 1-4 gauges on projected and unprojected columns,
   until at least N_CASES cases ran.

In both, every other output equals the exact reference of the query without gauges, a gauge's n equals the operand's
COUNT and its points are valid exactly where that COUNT is > 0, and the outputs are byte-identical across two runs."""
import copy

import numpy as np
import pytest

from cnosdb_b200.engine import PushedAggregate, Engine
from tests import sweep_reference as sw
from tests.gauge_reference import check_gauge, exact_gauge_cells
from tests.mode_reference import check_distinct, check_mode, exact_mode_cells
from tests.test_gpu_kernel_sweep import assert_same_bytes, check_exact, check_operands, prepared_run, scan_kwargs, set_env
from tests.test_gpu_mode_sweep import add_modes

pytestmark = pytest.mark.gpu

BASE_SEED = 20261019
N_CASES = 120


@pytest.fixture(scope="module")
def engine():
    e = Engine(0)
    yield e
    e.close()


def without(q, attrs):
    """q without the pseudo-aggregates `attrs`: entries that ask for nothing else are dropped, the others lose them."""
    q0 = copy.copy(q)
    cols = []
    for c in q.columns:
        if not any(getattr(c, a, False) for a in attrs):
            cols.append(c)
        elif c.agg_mask or any(getattr(c, a, False) for a in ("median", "increase", "mode", "count_distinct", "gauge_agg")
                               if a not in attrs):
            c2 = copy.copy(c)
            for a in attrs:
                setattr(c2, a, False)
            cols.append(c2)
    q0.columns, q0._keep = cols, None
    return q0


def check_case(got, truth, q, extra, what, tombstones=None, files=None):
    q0 = without(q, ("gauge_agg", "mode", "count_distinct"))
    exp = sw.expected(truth, q0, extra, tombstones=tombstones, files=files)
    assert not isinstance(exp, (int, str)), "%s: the reference refuses the query without gauges (%s)" % (what, exp)
    n0 = len(q0.output_names())
    assert got.names[:n0] == q0.output_names(), what
    head = copy.copy(got)
    head.names, head.values, head.validity = got.names[:n0], got.values[:n0], got.validity[:n0]
    if hasattr(exp, "pairs"):
        check_operands(head, exp, q0, what)
    else:
        check_exact(head, exp, what)
    n_cells = got.n_groups * got.n_buckets
    kw = dict(tombstones=tombstones, files=files, group_ids=extra.get("group_ids"), edges=extra.get("edges"),
              labels=extra.get("labels"))
    q1 = without(q, ("gauge_agg",))
    n1 = len(q1.output_names())
    assert got.names[:n1] == q1.output_names(), what
    for c, j in zip([c for c in q1.columns if c.mode] + [c for c in q1.columns if c.count_distinct],
                    range(n0, n1)):
        exact = exact_mode_cells(truth, q, c.column_id, c.phys_type, n_cells, **kw)
        (check_mode if got.names[j][1] == "mode" else check_distinct)(got, j, exact, what="%s %s" % (what, got.names[j]))
    gauges = [c for c in q.columns if c.gauge_agg]
    assert len(got.names) == n1 + 9 * len(gauges), what
    for k, c in enumerate(gauges):
        j0 = n1 + 9 * k
        assert got.names[j0] == (c.column_id, "gauge_n"), what
        check_gauge(got, j0, exact_gauge_cells(truth, q, c.column_id, c.phys_type, n_cells, **kw),
                    what="%s gauge %d of %d" % (what, k, c.column_id))
        if (c.column_id, "count") in got.names:
            count = got.values[got.names.index((c.column_id, "count"))]
            np.testing.assert_array_equal(got.values[j0], count, err_msg="%s: gauge n of %d != COUNT" % (what, c.column_id))
            for f in range(1, 9):
                bad = np.nonzero(got.validity[j0 + f] != (count > 0))[0]
                assert bad.size == 0, "%s: gauge of %d: validity differs from COUNT > 0 at %s" % (what, c.column_id, bad[:5])


def add_gauges(q, truth, rng):
    """1-4 gauges of the arena's numeric columns: on a projected entry or as entries of their own, sometimes twice on one
    column. False (nothing added) when the arena has no numeric column."""
    num = [c for c in sw.columns_of(truth) if sw.COLUMNS[c] != sw.BOOL]
    if not num:
        return False
    for _ in range(int(rng.integers(1, 5))):
        c = int(rng.choice(num))
        entry = [e for e in q.columns if e.column_id == c and e.agg_mask and not e.gauge_agg]
        if entry and rng.random() < 0.5:
            entry[0].gauge_agg = True
        else:
            q.columns.append(PushedAggregate(c, sw.COLUMNS[c], ["gauge_agg"]))
    return True


def test_every_bin(engine, monkeypatch):
    set_env(monkeypatch, {"TSKV_PARTS": None, "TSKV_SMEM_TABLE_KB": None})
    for b in range(sw.N_BINS):
        tk, vk = divmod(sw.serial_bin(b), sw.N_VK)
        s8b = vk == sw.VK_S8B and tk != sw.TK_GEN
        for narrow in ((sw.NARROW_NONE, sw.NARROW_SOME, sw.NARROW_ALL) if s8b else (sw.NARROW_NONE,)):
            arena, descs, truth = sw.bin_arena(b, narrow)
            for edges in (False, True):
                q, extra = sw.targeted_query(truth, (sw.SCAN, tk, vk, False, narrow, edges), seed=b)
                num = [c for c in sw.columns_of(truth) if sw.COLUMNS[c] != sw.BOOL]
                q.columns += [PushedAggregate(c, sw.COLUMNS[c], ["gauge_agg"]) for c in num]
                q.columns.append(PushedAggregate(num[0], sw.COLUMNS[num[0]], ["gauge_agg"]))
                what = "gauges in bin %d narrow %d edges %s" % (b, narrow, edges)
                pages = engine.upload_pages(arena, descs)
                try:
                    got, wl = prepared_run(engine, pages, q, extra)
                    assert wl is not None, "%s: status %s" % (what, got)
                    check_case(got, truth, q, extra, what)
                    again, _ = prepared_run(engine, pages, q, extra)
                    assert_same_bytes(got, again, what)
                    field = (descs["phys_type"] != 0) & np.isin(descs["series_id"], q.series_ids)
                    for c in num:
                        assert (wl["page_bin"][field & (descs["column_id"] == c)] == b).all(), what
                finally:
                    pages.close()


def test_random_combinations(engine, monkeypatch):
    ran, n_ops, outcomes, i = 0, 0, {}, 0
    while ran < N_CASES:
        assert i < 4 * N_CASES, "too few random cases take gauges: %d of %d" % (ran, i)
        case = sw.random_operand_case(i, BASE_SEED)
        i += 1
        base = sw.case_expected(case)
        rng = np.random.default_rng([BASE_SEED, i, 11])
        if isinstance(base, (int, str)) or "slide" in case.extra or not add_gauges(case.query, case.truth, rng):
            outcomes["skipped"] = outcomes.get("skipped", 0) + 1
            continue
        if rng.random() < 0.4:
            add_modes(case.query, case.truth, rng)
        n_ops += len([c for c in case.query.columns if c.gauge_agg])
        what = case.describe()
        set_env(monkeypatch, case.env)
        pages = engine.upload_pages(case.arena, case.descs, host_resident=case.host_resident, verify_on_read=case.verify_on_read)
        try:
            if case.tombstones is not None:
                pages.set_tombstones(case.tombstones)
            if case.files is not None:
                pages.set_chunk_files(case.files)
            got, wl = prepared_run(engine, pages, case.query, case.extra)
            assert wl is not None, "%s\nstatus %s, expected a result" % (what, got)
            check_case(got, case.truth, case.query, case.extra, what, tombstones=case.tombstones, files=case.files)
            again = engine.scan_aggregate(pages, case.query, **scan_kwargs(case.extra))
            assert_same_bytes(got, again, what)
        finally:
            pages.close()
        ran += 1
        shape = case.desc.get("grouping", "?")
        outcomes[shape] = outcomes.get(shape, 0) + 1
    print("\nrandom gauge combinations: %d cases with %d gauges over %d drawn; %s" % (ran, n_ops, i, outcomes))
