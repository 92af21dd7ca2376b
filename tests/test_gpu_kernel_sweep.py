"""Every instantiation of the fused scan's kernels, and random combinations of query features, against the exact reference.

1. test_every_instantiation: one case aimed at each key of sweep_reference.INSTANTIATIONS (k_scan_aggregate<TK, VK, SEL,
   NARROW, EDGES> and k_scan_m2<TK, VK, EDGES>) through its long bin, and through its short bin too where it runs one
   (bins 9-12). The arena holds field pages of that one bin only; the work list read back after the pass proves the bin
   held them with the intended narrow flag, so a change of the generator cannot move a case to another kernel unseen. The
   result is held to the exact reference (M2 to the exact M2), and the keys reached must be the whole list.
2. test_random_combinations: N_RANDOM seeded cases (tests/sweep_reference.py: random_case) that draw the arena's codecs,
   page lengths, NULLs, column groups and overlapping chunk files, the grouping (bucket, series, tags, edges, labels,
   sliding window, unbucketed), aggregates with FIRST / LAST and M2, predicates, time ranges, tombstones, a host-resident
   page set, CRC on read, TSKV_PARTS and TSKV_SMEM_TABLE_KB. Each is checked against its expected result or status, and
   scanned twice (a prepared scan, then an end-to-end call): every output that does not depend on the order of f64
   additions must be byte-identical. TSKV_SWEEP_CASE=<index> reruns one case.
3. test_random_operand_combinations: N_OPERAND random cases with column pairs and medians (sweep_reference:
   random_operand_case). Where the query projects COUNT(c), the pair (c, c)'s n and the median of c's validity must
   equal it first (the pairs' and medians' row selection against pass 1's); then the pairs by check_pair, the medians
   bit for bit and every other output against the exact reference, and medians and pair n byte-identical between two
   runs.
   TSKV_SWEEP_CASE=<index> reruns one case here too.
4. test_operands_in_every_bin: pairs over every numeric column pair and a median per numeric column over the arena of
   each bin (simple8b-value bins: wide, mixed and narrow pages), tumbling and edge scans; the work list read back proves
   the operands' pages sat in that bin's intended bucket.
   Each bin also runs a GROUP BY series copy of the query with an increase of every numeric column and one duplicate.
5. test_random_increase_combinations: N_INCREASE random cases with counter increases (sweep_reference:
   random_increase_case), most regrouped into a shape whose cells hold one series, the rest kept and held to the
   refusal rule of sweep_reference.increase_status. Where the query projects COUNT(c), each increase of c must be valid
   exactly where COUNT(c) > 0; then the increases by check_increase, and integer increases byte-identical between two
   runs. TSKV_SWEEP_CASE=<index> reruns one case here too.
6. test_every_operand_kernel_reached: tests 3, 4 and 5 together launched every operand kernel
   (sweep_reference.OPERAND_KERNELS) on work (skipped unless all three ran to the end, tests 3 and 5 over every
   case)."""
import copy
import os

import numpy as np
import pytest

from cnosdb_b200 import cabi
from cnosdb_b200.engine import PushedAggregate, TskvError
from tests import sweep_reference as sw
from tests.covariance_reference import check_pair
from tests.helpers import assert_matches_exact
from tests.increase_reference import check_increase
from tests.median_reference import check_median
from tests.variance_reference import check_m2

pytestmark = pytest.mark.gpu

BASE_SEED = 20261017
N_RANDOM = 300
N_OPERAND = 200
N_INCREASE = 150
ONE_CASE = os.environ.get("TSKV_SWEEP_CASE")  # rerun one index of test_random_combinations / _operand_combinations


class _Picked:
    """The outputs `keep` of a ScanResult / ExactResult (assert_matches_exact reads names, values, validity, phys and,
    for ExactResult, center / bound by output index)."""

    def __init__(self, res, keep):
        self.names = [res.names[j] for j in keep]
        self.values, self.validity, self.phys = res.values[keep], res.validity[keep], res.phys
        if hasattr(res, "center"):
            self.center = {i: res.center[j] for i, j in enumerate(keep) if j in res.center}
            self.bound = {i: res.bound[j] for i, j in enumerate(keep) if j in res.bound}


def check_exact(got, exp, what):
    """Every output against the exact reference: M2 by check_m2, the rest by assert_matches_exact."""
    rest = [j for j, (_, a) in enumerate(got.names) if a != "m2"]
    if len(rest) < len(got.names):
        check_m2(got, exp, what)
    assert_matches_exact(_Picked(got, rest), _Picked(exp, rest), what=what)


def deterministic_outputs(res):
    """Indices of the outputs that do not depend on the order of f64 additions: counts, integer sums and means, MIN /
    MAX and FIRST / LAST of every type, pair n, medians and integer increases."""
    return [j for j, (c, a) in enumerate(res.names)
            if not (a in ("m2", "c", "m2x", "m2y") or
                    (a in ("sum", "mean", "increase") and res.phys[c] == cabi.TSKV_PT_F64))]


def assert_same_bytes(a, b, what):
    keep = deterministic_outputs(a)
    assert a.names == b.names
    assert (a.validity == b.validity).all(), "%s: validity differs between two runs" % what
    bad = [a.names[j] for j in keep if (a.values[j] != b.values[j]).any()]
    assert not bad, "%s: outputs %s differ between two runs" % (what, bad)


def set_env(monkeypatch, env):
    for k, v in env.items():
        if v is None:
            monkeypatch.delenv(k, raising=False)
        else:
            monkeypatch.setenv(k, v)


def scan_kwargs(extra):
    return {k: extra[k] for k in ("slide", "group_ids", "n_groups", "edges", "labels") if k in extra}


def prepared_run(engine, pages, query, extra):
    """-> (ScanResult, work list) of a prepared scan, or (status, None) when the library refuses it."""
    try:
        scan = engine.prepare(pages, query, **scan_kwargs(extra))
    except TskvError as e:
        return e.status, None
    except ValueError:
        return "ValueError", None
    try:
        scan.run()
        return scan.finalize(), scan.work_list()
    except TskvError as e:
        return e.status, None
    finally:
        scan.close()


# ---- 1. every instantiation --------------------------------------------------------------------------------------------
def targets():
    """(key, bin) of every targeted case: the key's serial bin, and the short bin that runs the same kernels."""
    short_of = {s: b for b, s in sw.SHORT_BINS.items()}
    out = []
    for key in sw.INSTANTIATIONS:
        sb = key[1] * sw.N_VK + key[2]
        out.append((key, sb))
        if sb in short_of:
            out.append((key, short_of[sb]))
    return out


def arena_narrow(key):
    """The narrow flag the case's bin must carry: the key's, for the narrow variants; wide pages otherwise."""
    return key[4]


def test_every_instantiation(engine, monkeypatch):
    set_env(monkeypatch, {"TSKV_PARTS": None, "TSKV_SMEM_TABLE_KB": None})
    reached, short_reached, arenas = {}, set(), {}
    for i, (key, b) in enumerate(targets()):
        what = "%s via bin %d" % (sw.key_name(key), b)
        narrow = arena_narrow(key)
        if (b, narrow) not in arenas:
            arenas[(b, narrow)] = sw.bin_arena(b, narrow)
        arena, descs, truth = arenas[(b, narrow)]
        q, extra = sw.targeted_query(truth, key, seed=i)
        exp = sw.expected(truth, q, extra)
        assert not isinstance(exp, (int, str)), "%s: the reference refuses the case (%s)" % (what, exp)
        pages = engine.upload_pages(arena, descs)
        try:
            got, wl = prepared_run(engine, pages, q, extra)
        finally:
            pages.close()
        assert wl is not None, "%s: status %s" % (what, got)
        field = (descs["phys_type"] != cabi.TSKV_PT_TIME) & np.isin(descs["series_id"], q.series_ids)
        assert (wl["page_bin"][field] == b).all(), "%s: field pages in bins %s" % (what, sorted(set(wl["page_bin"][field])))
        assert sw.bin_fill(wl, len(q.columns))[b].sum() == field.sum(), what
        flags = sw.bin_narrow_flags(wl, descs)
        assert flags[b] == narrow, "%s: narrow flag %d" % (what, flags[b])
        if narrow != sw.NARROW_SOME and sw.serial_bin(b) in (0, 3):  # (HELPER_SERIES)
            assert sw.NARROW_SOME in flags, "%s: the work list reports no narrow flags" % what
        keys = sw.kernel_keys(wl, descs, q, "edges" in extra)
        assert key in keys and all(bins == {b} for bins in keys.values()), "%s: ran %s" % (what, keys)
        check_exact(got, exp, what)
        for k in keys:
            reached.setdefault(k, set()).add(b)
        if b >= sw.N_SERIAL_BINS:
            short_reached.add(b)
    missed = [sw.key_name(k) for k in sw.INSTANTIATIONS if k not in reached]
    assert not missed, "instantiations no targeted case reached: %s" % missed
    assert short_reached == set(sw.SHORT_BINS), short_reached
    print("\nkernel sweep: %d of %d instantiations reached, short bins %s" % (len(reached), len(sw.INSTANTIATIONS),
                                                                           sorted(short_reached)))


def check_operands(got, exp, query, what):
    """The pairs, medians and increases of `got` against exp.pairs / exp.medians / exp.increases
    (sweep_reference.expected), and every other output against the rest of exp. First, where the query projects
    COUNT(c): the pair (c, c)'s n equals it, and the median of c and every increase of c are valid where it is > 0."""
    meds = [c for c in query.columns if c.median]
    incs = [c for c in query.columns if c.increase]
    i0 = len(got.names) - len(incs)  # (the increase outputs come last, in column order)
    m0 = i0 - len(meds)  # (the median outputs come before them, in column order)
    assert got.names[m0:] == [(c.column_id, "median") for c in meds] + [(c.column_id, "increase") for c in incs], what
    for k, (x, _, y, _) in enumerate(query.pairs):
        if x == y and (x, "count") in got.names:
            n, _ = got.pair(k, "n")
            count = got.values[got.names.index((x, "count"))]
            bad = np.nonzero(n.ravel() != count)[0]
            assert bad.size == 0, "%s: pair %d (%d, %d): n differs from COUNT at cells %s: the selection passes " \
                "disagree with pass 1" % (what, k, x, x, bad[:5])
    for k, c in enumerate(meds):
        if (c.column_id, "count") in got.names:
            count = got.values[got.names.index((c.column_id, "count"))]
            bad = np.nonzero(got.validity[m0 + k] != (count > 0))[0]
            assert bad.size == 0, "%s: median %d of %d: validity differs from COUNT > 0 at cells %s: the selection " \
                "passes disagree with pass 1" % (what, k, c.column_id, bad[:5])
    for k, c in enumerate(incs):
        if (c.column_id, "count") in got.names:
            count = got.values[got.names.index((c.column_id, "count"))]
            bad = np.nonzero(got.validity[i0 + k] != (count > 0))[0]
            assert bad.size == 0, "%s: increase %d of %d: validity differs from COUNT > 0 at cells %s: the increase " \
                "pass disagrees with pass 1" % (what, k, c.column_id, bad[:5])
    for k in range(len(query.pairs)):
        check_pair(got, k, exp.pairs[k], what="%s pair %d" % (what, k))
    for k in range(len(meds)):
        check_median(got, m0 + k, exp.medians[k], what="%s median %d" % (what, k))
    for k, c in enumerate(incs):
        check_increase(got, i0 + k, exp.increases[k], c.phys_type, what="%s increase %d of %d" % (what, k, c.column_id))
    rest = list(range(m0 - 4 * len(query.pairs)))
    assert got.names[:len(rest)] == exp.names[:len(rest)], what
    check_exact(_Picked(got, rest), _Picked(exp, rest), what)


# ---- 2. random combinations --------------------------------------------------------------------------------------------
def run_case(engine, case, exp, monkeypatch, reached_operands=None):
    """-> the instantiation keys the case ran; adds the operand kernels it launched on work to reached_operands. Fails
    with the case's description."""
    what = case.describe()
    set_env(monkeypatch, case.env)
    pages = engine.upload_pages(case.arena, case.descs, host_resident=case.host_resident,
                                verify_on_read=case.verify_on_read)
    try:
        if case.tombstones is not None:
            pages.set_tombstones(case.tombstones)
        if case.files is not None:
            pages.set_chunk_files(case.files)
        got, wl = prepared_run(engine, pages, case.query, case.extra)
        if isinstance(exp, (int, str)):
            assert got == exp, "%s\nstatus %s, expected %s" % (what, got, exp)
            return {}
        assert wl is not None, "%s\nstatus %s, expected a result" % (what, got)
        if hasattr(exp, "pairs"):
            check_operands(got, exp, case.query, what)
            reached_operands |= sw.operand_kernels(wl, case.query, "edges" in case.extra, case.truth, case.files)
        else:
            check_exact(got, exp, what)
        again = engine.scan_aggregate(pages, case.query, **scan_kwargs(case.extra))
        assert_same_bytes(got, again, what)
        return sw.kernel_keys(wl, case.descs, sw.scan_query(case.query), "edges" in case.extra)
    finally:
        pages.close()


def test_random_combinations(engine, monkeypatch):
    indices = [int(ONE_CASE)] if ONE_CASE is not None else range(N_RANDOM)
    reached, statuses = {}, {}
    for i in indices:
        case = sw.random_case(i, BASE_SEED)
        exp = sw.case_expected(case)
        outcome = exp if isinstance(exp, (int, str)) else "result"
        statuses[outcome] = statuses.get(outcome, 0) + 1
        for k, bins in run_case(engine, case, exp, monkeypatch).items():
            reached.setdefault(k, set()).update(bins)
    short = sorted({b for bins in reached.values() for b in bins if b >= sw.N_SERIAL_BINS})
    print("\nrandom combinations: %d cases, outcomes %s, %d of %d instantiations reached, short bins %s; not reached: %s" % (
        len(indices), statuses, len(reached), len(sw.INSTANTIATIONS), short,
        [sw.key_name(k) for k in sw.INSTANTIATIONS if k not in reached]))


# ---- 3. random combinations with pairs and medians -------------------------------------------------------------------
OPERANDS_REACHED = set()  # the operand kernels tests 3, 4 and 5 launched on work
OPERAND_TESTS_RUN = set()  # tests 3 (every case), 4 and 5 (every case) when they ran to the end in this session


def test_random_operand_combinations(engine, monkeypatch):
    indices = [int(ONE_CASE)] if ONE_CASE is not None else range(N_OPERAND)
    statuses, n_pairs, n_meds = {}, 0, 0
    for i in indices:
        case = sw.random_operand_case(i, BASE_SEED)
        exp = sw.case_expected(case)
        outcome = exp if isinstance(exp, (int, str)) else "result"
        statuses[outcome] = statuses.get(outcome, 0) + 1
        n_pairs += len(case.query.pairs)
        n_meds += len([c for c in case.query.columns if c.median])
        run_case(engine, case, exp, monkeypatch, OPERANDS_REACHED)
    if ONE_CASE is None:
        OPERAND_TESTS_RUN.add("random")
    print("\nrandom operand combinations: %d cases, %d pairs, %d medians, outcomes %s; operand kernels reached: %s" % (
        len(indices), n_pairs, n_meds, statuses, sorted(OPERANDS_REACHED)))


# ---- 4. operands in every bin ----------------------------------------------------------------------------------------
def operand_query(truth, b, narrow, edges):
    """targeted_query's tumbling or edge query of bin b's arena, plus a pair of every two numeric columns (x == y too)
    and a median of every numeric column."""
    tk, vk = divmod(sw.serial_bin(b), sw.N_VK)
    q, extra = sw.targeted_query(truth, (sw.SCAN, tk, vk, False, narrow, edges), seed=b)
    num = [c for c in sw.columns_of(truth) if sw.COLUMNS[c] != sw.BOOL]
    q.pairs = [(x, sw.COLUMNS[x], y, sw.COLUMNS[y]) for i, x in enumerate(num) for y in num[i:]]
    q.columns += [PushedAggregate(c, sw.COLUMNS[c], ["median"]) for c in num]
    return q, extra, num


def increase_query(q, num):
    """A GROUP BY series copy of operand_query's query without its pairs and medians, plus an increase of every numeric
    column and a second increase of the first."""
    qi = copy.copy(q)
    qi.pairs, qi._keep, qi.group_by_series = [], None, True
    qi.columns = [c for c in q.columns if not c.median] + \
        [PushedAggregate(c, sw.COLUMNS[c], ["increase"]) for c in num + num[:1]]
    return qi


def operand_bin_case(engine, arena, descs, truth, q, extra, b, narrow, num, what):
    """Runs one query of test_operands_in_every_bin -> (work list, the buckets its operands' items sat in)."""
    exp = sw.expected(truth, q, extra)
    assert not isinstance(exp, (int, str)), "%s: the reference refuses the case (%s)" % (what, exp)
    pages = engine.upload_pages(arena, descs)
    try:
        got, wl = prepared_run(engine, pages, q, extra)
    finally:
        pages.close()
    assert wl is not None, "%s: status %s" % (what, got)
    # every page of every operand in bin b, in the wide or the narrow bucket as its narrow flag says
    ids = [c.column_id for c in sw.scan_query(q).columns]
    fill = wl["fill"].astype(np.int64).reshape(sw.N_BINS, len(ids), 2)
    field = (descs["phys_type"] != cabi.TSKV_PT_TIME) & np.isin(descs["series_id"], q.series_ids)
    buckets = set()
    for c in num:
        mine = field & (descs["column_id"] == c)
        nar = int(wl["page_narrow"][mine].astype(bool).sum())
        qc = ids.index(c)
        assert (wl["page_bin"][mine] == b).all() and fill[:, qc].sum() == fill[b, qc].sum(), what
        assert (fill[b, qc, 0], fill[b, qc, 1]) == (int(mine.sum()) - nar, nar), (what, c, fill[b, qc])
        if narrow == sw.NARROW_ALL:
            assert fill[b, qc, 0] == 0 and fill[b, qc, 1] > 0, (what, c, fill[b, qc])
        buckets |= {k for k in (0, 1) if fill[b, qc, k]}
    check_operands(got, exp, q, what)
    return wl, buckets


def test_operands_in_every_bin(engine, monkeypatch):
    set_env(monkeypatch, {"TSKV_PARTS": None, "TSKV_SMEM_TABLE_KB": None})
    reached, buckets = set(), set()
    for b in range(sw.N_BINS):
        tk, vk = divmod(sw.serial_bin(b), sw.N_VK)
        s8b = vk == sw.VK_S8B and tk != sw.TK_GEN  # (the bins whose pages the scan keeps in a narrow bucket)
        for narrow in ((sw.NARROW_NONE, sw.NARROW_SOME, sw.NARROW_ALL) if s8b else (sw.NARROW_NONE,)):
            arena, descs, truth = sw.bin_arena(b, narrow)
            for edges in (False, True):
                q, extra, num = operand_query(truth, b, narrow, edges)
                what = "operands in bin %d narrow %d edges %s" % (b, narrow, edges)
                wl, bk = operand_bin_case(engine, arena, descs, truth, q, extra, b, narrow, num, what)
                buckets |= bk
                reached |= sw.operand_kernels(wl, q, edges)
                qi = increase_query(q, num)
                wl, bk = operand_bin_case(engine, arena, descs, truth, qi, extra, b, narrow, num, what + " increases")
                buckets |= bk
                reached |= sw.operand_kernels(wl, qi, edges)
    assert buckets == {0, 1}, buckets
    OPERANDS_REACHED.update(reached)
    OPERAND_TESTS_RUN.add("bins")
    print("\noperands in every bin: operand kernels reached: %s" % sorted(reached))


# ---- 5. random combinations with increases ---------------------------------------------------------------------------
def test_random_increase_combinations(engine, monkeypatch):
    indices = [int(ONE_CASE)] if ONE_CASE is not None else range(N_INCREASE)
    statuses, shapes, n_incs = {}, {}, 0
    for i in indices:
        case = sw.random_increase_case(i, BASE_SEED)
        exp = sw.case_expected(case)
        outcome = exp if isinstance(exp, (int, str)) else "result"
        statuses[outcome] = statuses.get(outcome, 0) + 1
        shape = "%s -> %s" % (case.desc["shape"], outcome)
        shapes[shape] = shapes.get(shape, 0) + 1
        n_incs += len([c for c in case.query.columns if c.increase])
        run_case(engine, case, exp, monkeypatch, OPERANDS_REACHED)
    if ONE_CASE is None:
        OPERAND_TESTS_RUN.add("increases")
    print("\nrandom increase combinations: %d cases, %d increases, outcomes %s, shapes %s; operand kernels reached: %s"
          % (len(indices), n_incs, statuses, shapes, sorted(OPERANDS_REACHED)))


def test_every_operand_kernel_reached():
    """Tests 3, 4 and 5 together launched every operand kernel on work. It reads what they recorded, so it needs all
    three to have run to the end in this session, tests 3 and 5 over every case; otherwise it is skipped and says so."""
    if OPERAND_TESTS_RUN != {"random", "bins", "increases"}:
        pytest.skip("needs test_random_operand_combinations (every case), test_operands_in_every_bin and "
                    "test_random_increase_combinations (every case) to run first in this session; ran: %s"
                    % sorted(OPERAND_TESTS_RUN))
    missed = [k for k in sw.OPERAND_KERNELS if k not in OPERANDS_REACHED]
    assert not missed, "operand kernels no operand test launched on work: %s" % missed
    print("\noperand kernels reached: %s" % sorted(OPERANDS_REACHED))
