"""mode(x) and COUNT(DISTINCT x) over every fused-scan bin and over random query combinations, against
tests/mode_reference.py bit for bit:

1. test_every_bin: sweep_reference.bin_arena's arena of every bin (time class x value encoding; the simple8b bins with
   wide, mixed and narrow pages, the generic bin's short, run-length and all-NULL pages), tumbling and edge grids, with a
   mode and a distinct count of every numeric column (I64, U64, F64) and a second mode of the first. Every operand page
   sits in the bin, and the operand kernels launched on work.
2. test_random_combinations: seeded sweep_reference.random_operand_case cases (pairs, medians, tombstones, chunk files,
   predicates, host-resident and verify-on-read page sets, every grouping but sliding windows) with 1-4 mode and distinct
   operands added from a stream of their own, on projected and unprojected columns, until at least N_CASES cases ran.

In both, where the query projects COUNT(c), the mode of c is valid exactly where COUNT > 0 (the gather agrees with pass
1), every other output equals the exact reference of the query without modes and distincts, and the integer outputs
are byte-identical across two runs."""
import copy

import numpy as np
import pytest

from cnosdb_b200 import cabi
from cnosdb_b200.engine import Engine, PushedAggregate
from tests import sweep_reference as sw
from tests.mode_reference import check_distinct, check_mode, exact_mode_cells
from tests.test_gpu_kernel_sweep import assert_same_bytes, check_exact, check_operands, prepared_run, scan_kwargs, set_env

pytestmark = pytest.mark.gpu

BASE_SEED = 20261018
N_CASES = 120


@pytest.fixture(scope="module")
def engine():
    e = Engine(0)
    yield e
    e.close()


def without_modes(q):
    """q without its modes and distincts: entries that ask for nothing else are dropped, the others lose the flags."""
    q0 = copy.copy(q)
    cols = []
    for c in q.columns:
        if not (c.mode or c.count_distinct):
            cols.append(c)
        elif c.agg_mask or c.median or c.increase:
            c2 = copy.copy(c)
            c2.mode = c2.count_distinct = False
            cols.append(c2)
    q0.columns, q0._keep = cols, None
    return q0


def check_case(got, truth, q, extra, what, tombstones=None, files=None):
    """got against the exact reference (see the module docstring)."""
    q0 = without_modes(q)
    exp = sw.expected(truth, q0, extra, tombstones=tombstones, files=files)
    assert not isinstance(exp, (int, str)), "%s: the reference refuses the query without modes (%s)" % (what, exp)
    n0 = len(q0.output_names())
    assert got.names[:n0] == q0.output_names(), what
    head = copy.copy(got)
    head.names, head.values, head.validity = got.names[:n0], got.values[:n0], got.validity[:n0]
    if hasattr(exp, "pairs"):
        check_operands(head, exp, q0, what)
    else:
        check_exact(head, exp, what)
    modes = [c for c in q.columns if c.mode]
    dists = [c for c in q.columns if c.count_distinct]
    assert got.names[n0:] == [(c.column_id, "mode") for c in modes] + [(c.column_id, "count_distinct") for c in dists], what
    n_cells = got.n_groups * got.n_buckets
    kw = dict(tombstones=tombstones, files=files, group_ids=extra.get("group_ids"), edges=extra.get("edges"),
              labels=extra.get("labels"))
    cache = {}
    for k, c in enumerate(modes + dists):
        key = (c.column_id, c.phys_type)
        if key not in cache:
            cache[key] = exact_mode_cells(truth, q, c.column_id, c.phys_type, n_cells, **kw)
        j = n0 + k
        if k < len(modes):
            if (c.column_id, "count") in got.names:
                count = got.values[got.names.index((c.column_id, "count"))]
                bad = np.nonzero(got.validity[j] != (count > 0))[0]
                assert bad.size == 0, "%s: mode of %d: validity differs from COUNT > 0 at cells %s" % (what, c.column_id, bad[:5])
            check_mode(got, j, cache[key], what="%s mode %d of %d" % (what, k, c.column_id))
        else:
            check_distinct(got, j, cache[key], what="%s distinct %d of %d" % (what, k, c.column_id))


def add_modes(q, truth, rng):
    """1-4 modes / distincts of the arena's numeric columns: on a projected entry (it asks for them too) or as entries
    of their own, sometimes twice on one column. False (nothing added) when the arena has no numeric column."""
    num = [c for c in sw.columns_of(truth) if sw.COLUMNS[c] != sw.BOOL]
    if not num:
        return False
    for _ in range(int(rng.integers(1, 5))):
        c = int(rng.choice(num))
        kind = str(rng.choice(["mode", "count_distinct"]))
        entry = [e for e in q.columns if e.column_id == c and e.agg_mask and not getattr(e, kind)]
        if entry and rng.random() < 0.5:
            setattr(entry[0], kind, True)
        else:
            q.columns.append(PushedAggregate(c, sw.COLUMNS[c], [kind]))
    return True


def test_every_bin(engine, monkeypatch):
    set_env(monkeypatch, {"TSKV_PARTS": None, "TSKV_SMEM_TABLE_KB": None})
    buckets = set()
    for b in range(sw.N_BINS):
        tk, vk = divmod(sw.serial_bin(b), sw.N_VK)
        s8b = vk == sw.VK_S8B and tk != sw.TK_GEN
        for narrow in ((sw.NARROW_NONE, sw.NARROW_SOME, sw.NARROW_ALL) if s8b else (sw.NARROW_NONE,)):
            arena, descs, truth = sw.bin_arena(b, narrow)
            for edges in (False, True):
                q, extra = sw.targeted_query(truth, (sw.SCAN, tk, vk, False, narrow, edges), seed=b)
                num = [c for c in sw.columns_of(truth) if sw.COLUMNS[c] != sw.BOOL]
                q.columns += [PushedAggregate(c, sw.COLUMNS[c], ["mode", "count_distinct"]) for c in num]
                q.columns.append(PushedAggregate(num[0], sw.COLUMNS[num[0]], ["mode"]))
                what = "modes in bin %d narrow %d edges %s" % (b, narrow, edges)
                pages = engine.upload_pages(arena, descs)
                try:
                    got, wl = prepared_run(engine, pages, q, extra)
                    assert wl is not None, "%s: status %s" % (what, got)
                    check_case(got, truth, q, extra, what)
                    again, _ = prepared_run(engine, pages, q, extra)
                    assert_same_bytes(got, again, what)
                finally:
                    pages.close()
                # every page of every operand sits in bin b, in the wide or the narrow bucket as its flag says
                ids = [c.column_id for c in q.projected()]
                ids += [c.column_id for c in q.columns if (c.mode or c.count_distinct) and c.column_id not in ids]
                fill = wl["fill"].astype(np.int64).reshape(sw.N_BINS, -1, 2)
                field = (descs["phys_type"] != cabi.TSKV_PT_TIME) & np.isin(descs["series_id"], q.series_ids)
                for c in num:
                    mine = field & (descs["column_id"] == c)
                    nar = int(wl["page_narrow"][mine].astype(bool).sum())
                    qc = ids.index(c)
                    assert (wl["page_bin"][mine] == b).all(), what
                    assert (fill[b, qc, 0], fill[b, qc, 1]) == (int(mine.sum()) - nar, nar), (what, c, fill[b, qc])
                    buckets |= {k for k in (0, 1) if fill[b, qc, k]}
    assert buckets == {0, 1}, buckets


def test_random_combinations(engine, monkeypatch):
    ran, n_ops, outcomes, i = 0, 0, {}, 0
    while ran < N_CASES:
        assert i < 4 * N_CASES, "too few random cases take modes: %d of %d" % (ran, i)
        case = sw.random_operand_case(i, BASE_SEED)
        i += 1
        base = sw.case_expected(case)
        # (a refused case, or one without a numeric column: modes add nothing to test)
        if isinstance(base, (int, str)) or "slide" in case.extra or \
                not add_modes(case.query, case.truth, np.random.default_rng([BASE_SEED, i, 7])):
            outcomes["skipped"] = outcomes.get("skipped", 0) + 1
            continue
        n_ops += len([c for c in case.query.columns if c.mode]) + len([c for c in case.query.columns if c.count_distinct])
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
    print("\nrandom mode combinations: %d cases with %d modes / distincts over %d drawn; %s" % (ran, n_ops, i, outcomes))
