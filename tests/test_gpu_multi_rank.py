"""The multi-rank merge at one to eight ranks (tests/ranks.py: every rank's series shard scanned as its own page set with
the global query, then merged through the all-gather merge and through the all-reduce partials path).

Every query family runs through every layout of tests/ranks.layouts (contiguous, id % N, uneven, a rank holding only
unselected series, a rank with no page, reversed gather order) at N = 1, 3, 4 and 8, and every case checks that
  - every rank exchanges the same number of words, and every rank's finalized result is the same, byte for byte;
  - the result matches the exact reference (M2 within its tolerance);
  - an integer MEAN equals the rank-order value bit for bit: each rank's exact sum rounded once to f64, added in gather
    order from +0.0, over the count (ranks.rank_order_mean);
  - the all-reduce path gives the gather path's result byte for byte (M2 scans refuse tskvgpu_scan_partials);
  - one rank is a no-op: N = 1 gives the plain finalize of the same pass (NaN as NaN);
  - the reader counters of the ranks add up to those of the whole scan;
  - reversed gather order changes nothing but f64 SUM, MEAN (integer MEAN too) and M2.
Families: tumbling ALL aggregates on i64 / u64 / f64 / bool with NULLs, ungrouped and by series; unbucketed FIRST /
LAST over clipped ranges on ranks whose time minima differ; ranges, predicates, tombstones and the overlap merge;
edges with FIRST / LAST, labels, GROUP BY tags; sliding windows; M2 with COUNT and MEAN; TSKV_PARTS=3 and
TSKV_SMEM_TABLE_KB=0; column pairs (covar / corr) with COUNT and MEAN. M2 arenas of their own put the between-rank term,
means near 2^63, ill-conditioned cells and special values through k_merge_m2 at the rank count that splits their cells,
and the same arenas put the first three through k_merge_pairs.
M2 and pair scans refuse tskvgpu_scan_partials; their moments are held to the exact ones within a tolerance, and the
one-rank merge of a pair's moments (Chan's formulas around the rank's own means) to them, not to the plain finalize's
bytes."""
import copy
import functools
import math

import numpy as np
import pytest

from cnosdb_b200 import cabi, datagen
from cnosdb_b200.engine import PushedAggregate, QueryOption, TskvError
from tests import exact_arenas as ea
from tests.edges_reference import exact_aggregate_edges
from tests.group_reference import exact_aggregate_grouped
from tests.covariance_reference import check_pair, exact_pair_cells
from tests.helpers import assert_matches_exact, bucket_spec, exact_aggregate
from tests.labels_reference import exact_aggregate_labels
from tests.ranks import RankScans, layouts, rank_order_mean
from tests.sliding_reference import expand_aggregate, sliding_fit_grid
from tests.test_gpu_bucket_edges import edge_query, random_edges, span
from tests.test_gpu_bucket_labels import label_query
from tests.variance_reference import check_m2, exact_m2, with_m2

pytestmark = pytest.mark.gpu

NS = (1, 3, 4, 8)
COUNTERS = ("points_decoded", "rows_in_range", "page_read_count", "page_read_bytes", "pruned_page_count")
I64, F64, U64, BOOL = cabi.TSKV_PT_I64, cabi.TSKV_PT_F64, cabi.TSKV_PT_U64, cabi.TSKV_PT_BOOL
FIELDS = ((1, I64), (2, F64), (3, U64), (4, BOOL))
NUM = FIELDS[:3]
PLAIN = ("count", "sum", "min", "max", "mean")
M2_AGGS = ("count", "mean", "m2")
T0, STEP = 1_000_000, 1000
N_SERIES = 48
ALL_IDS = np.arange(N_SERIES, dtype=np.uint32)
SELECTED = ALL_IDS[ALL_IDS % 6 != 5]  # 40 series; the other 8 are never selected
UNSELECTED = ALL_IDS[ALL_IDS % 6 == 5]


# ---- families ----------------------------------------------------------------------------------------------------------
class Family:
    """One query over one arena: ref(truth, files) is the exact reference of the query over (a shard of) the arena; with
    m2_rtol the query holds M2 and the expected result gets its exact M2 (variance_reference.with_m2); with pair_rtol it
    holds column pairs, held to their exact co-moments (covariance_reference.exact_pair_cells)."""

    def __init__(self, name, arena, descs, truth, q, ref, prep=None, files=None, tombstones=None, env=None,
                 m2_rtol=None, unselected=(), all_ids=None, n_groups=None, pair_rtol=None):
        self.name, self.arena, self.descs, self.truth, self.ref = name, arena, descs, truth, ref
        self.q = q
        self.q.multi_rank = True
        self.prep = prep or {}
        self.files, self.tombstones, self.env, self.m2_rtol = files, tombstones, env or {}, m2_rtol
        self.pair_rtol = pair_rtol
        self._pairs = None
        self.unselected = unselected
        self.all_ids = np.asarray(sorted(truth) if all_ids is None else all_ids, dtype=np.uint32)
        self.n_groups = n_groups
        self._shard_refs = {}
        self._exp = None
        self._whole = None

    def expected(self):
        if self._exp is None:
            run = lambda: self.ref(self.truth, self.files)  # noqa: E731
            self._exp = with_m2(run, self.q, n_groups=self.n_groups) if self.m2_rtol else run()
        return self._exp

    def pairs(self):
        """exact_pair_cells of every pair of the query."""
        if self._pairs is None:
            n_cells = self.expected().values.shape[1]
            kw = dict(tombstones=self.tombstones, files=self.files)
            self._pairs = [exact_pair_cells(self.truth, self.q, p, n_cells, **kw) for p in self.q.pairs]
        return self._pairs

    def shard_ref(self, ids):
        """The exact reference over one shard's series (for its exact integer sums)."""
        key = tuple(int(i) for i in ids)
        if key not in self._shard_refs:
            keep, t, f, k = set(key), {}, [], 0
            for sid, cgs in self.truth.items():
                if sid in keep:
                    t[sid] = cgs
                    if self.files is not None:
                        f += list(self.files[k:k + len(cgs)])
                k += len(cgs)
            self._shard_refs[key] = self.ref(t, None if self.files is None else np.array(f, dtype=np.uint64))
        return self._shard_refs[key]

    def whole_counters(self, engine):
        """The reader counters of the same query scanned over the whole arena on one rank."""
        if self._whole is None:
            with RankScans(engine, self.arena, self.descs, self.q, [self.all_ids], files=self.files,
                           tombstones=self.tombstones, **self.prep) as rs:
                self._whole = rs.run()[0]
        return self._whole


def tumbling_arena(seed=1):
    """48 series of 40-200 rows, series sid starting 7 * sid steps after T0 (shards' time minima differ), every third one
    jittered; i64 / f64 / u64 / bool columns with 15 % NULLs, wide values in every fourth series."""
    rng = np.random.default_rng(seed)
    b = datagen.ArenaBuilder()
    truth = {}
    for sid in range(N_SERIES):
        n = int(rng.integers(40, 200))
        ts = T0 + (7 * sid + np.arange(n, dtype=np.int64)) * STEP
        if sid % 3 == 1:
            ts = ts + rng.integers(0, STEP // 2, n)
        fl, cols = [], {}
        for col, pt in FIELDS:
            vals = ea._values(rng, pt, n, wide=sid % 4 == 3)
            valid = rng.random(n) >= 0.15
            fl.append((col, pt, vals, None if valid.all() else valid))
            cols[col] = (vals, valid)
        b.add_column_group(sid, ts, fl)
        truth[sid] = [(ts, cols)]
    arena, descs = b.finish()
    return arena, descs, truth


def m2_arena(seed=2):
    rng = np.random.default_rng(seed)
    from tests.helpers import random_arena
    return random_arena(rng, n_series=N_SERIES, n_points=200, fields=NUM, null_frac=0.1, jitter=200, multi_cg=True)


def _grid(truth, width):
    lo, hi = span(truth)
    fbs, nb = bucket_spec(lo, hi, width)
    return dict(width=width, first_bucket_start=fbs, n_buckets=nb)


def _plain_ref(q):
    return lambda t, f: exact_aggregate(t, q)


FAMILIES = ("tumbling", "tumbling_by_series", "unbucketed_first_last", "filters", "edges", "labels", "tags", "sliding",
            "m2", "m2_by_series", "parts3", "smem0", "smem0_m2", "pairs")
PAIRS = [(1, I64, 2, F64), (2, F64, 3, U64), (3, U64, 3, U64), (2, F64, 1, I64)]


@functools.lru_cache(maxsize=None)
def family(name):
    if name == "filters":
        arena, descs, truth, files = ea.merge_arena()
        tombs = ea.merge_tombstones(truth)
        ids = np.arange(ea.MG_SERIES, dtype=np.uint32)
        sub = ids[ids % 5 != 2]
        fbs, nb = bucket_spec(ea.MG_T0 - ea.MG_W, ea.MG_T0 + 320 * ea.MG_STEP, ea.MG_W, origin=ea.MG_ORIGIN)
        ranges = [(ea.MG_T0 + 20 * ea.MG_STEP, ea.MG_T0 + 133 * ea.MG_STEP - 1),
                  (ea.MG_T0 + 180 * ea.MG_STEP + 1, ea.MG_T0 + 290 * ea.MG_STEP)]
        q = QueryOption(ea.sel_columns(ea.MG_FIELDS), series_ids=sub, time_ranges=ranges,
                        predicates=[(1, I64, ">", -2**40)], width=ea.MG_W, origin=ea.MG_ORIGIN, first_bucket_start=fbs,
                        n_buckets=nb)
        unselected = np.setdiff1d(np.array(sorted(truth), dtype=np.uint32), sub)
        return Family(name, arena, descs, truth, q, lambda t, f: exact_aggregate(t, q, tombstones=tombs, files=f),
                      files=files, tombstones=tombs, unselected=unselected)
    if name == "pairs":
        arena, descs, truth = m2_arena()
        q = QueryOption([PushedAggregate(c, pt, ("count", "mean")) for c, pt in NUM], series_ids=SELECTED, pairs=PAIRS,
                        **_grid(truth, 23_000))
        return Family(name, arena, descs, truth, q, _plain_ref(q), unselected=UNSELECTED, pair_rtol=1e-9)
    if name.startswith("m2") or name == "smem0_m2":
        arena, descs, truth = m2_arena()
        gbs = name == "m2_by_series"
        q = QueryOption([PushedAggregate(c, pt, M2_AGGS) for c, pt in NUM], series_ids=SELECTED, group_by_series=gbs,
                        **_grid(truth, 23_000))
        env = {"TSKV_SMEM_TABLE_KB": "0"} if name == "smem0_m2" else None
        return Family(name, arena, descs, truth, q, _plain_ref(q), env=env, m2_rtol=1e-9, unselected=UNSELECTED)
    arena, descs, truth = tumbling_arena()
    lo, hi = span(truth)
    cols = ea.sel_columns(FIELDS)
    grid = _grid(truth, 20_000)
    if name in ("tumbling", "tumbling_by_series", "parts3", "smem0"):
        q = QueryOption(cols, series_ids=SELECTED, group_by_series=name == "tumbling_by_series", **grid)
        env = {"parts3": {"TSKV_PARTS": "3"}, "smem0": {"TSKV_SMEM_TABLE_KB": "0"}}.get(name)
        return Family(name, arena, descs, truth, q, _plain_ref(q), env=env, unselected=UNSELECTED)
    if name == "unbucketed_first_last":
        mid = (lo + hi) // 2
        q = QueryOption(cols, series_ids=SELECTED, time_ranges=[(lo + 3_333, mid), (mid + 50_000, hi - 4_444)])
        return Family(name, arena, descs, truth, q, _plain_ref(q), unselected=UNSELECTED)
    if name == "edges":
        q, e = edge_query(QueryOption(cols, series_ids=SELECTED), random_edges(np.random.default_rng(3), lo, hi, 30, True))
        return Family(name, arena, descs, truth, q, lambda t, f: exact_aggregate_edges(t, q, e), prep={"edges": e},
                      unselected=UNSELECTED)
    if name == "labels":
        e = random_edges(np.random.default_rng(4), lo, hi, 40, True)
        lab = (np.arange(e.size - 1) % 6).astype(np.uint32)
        plain = [PushedAggregate(c, pt, ("count", "min", "max") if pt == BOOL else PLAIN) for c, pt in FIELDS]
        q = label_query(QueryOption(plain, series_ids=SELECTED), 6)
        return Family(name, arena, descs, truth, q, lambda t, f: exact_aggregate_labels(t, q, e, lab),
                      prep={"edges": e, "labels": lab}, unselected=UNSELECTED)
    if name == "tags":
        gid = (np.arange(SELECTED.size) * 7 % 5).astype(np.uint32)  # every group spans ranks
        q = QueryOption(cols, series_ids=SELECTED, **grid)
        return Family(name, arena, descs, truth, q, lambda t, f: exact_aggregate_grouped(t, q, gid, 5),
                      prep={"group_ids": gid, "n_groups": 5}, unselected=UNSELECTED, n_groups=5)
    assert name == "sliding"
    window, slide = 30_000, 10_000
    fbs, nb = sliding_fit_grid(truth, window, slide, 0, [])
    q = QueryOption([PushedAggregate(c, pt, PLAIN) for c, pt in NUM], series_ids=SELECTED, width=window,
                    first_bucket_start=fbs, n_buckets=nb)
    return Family(name, arena, descs, truth, q, lambda t, f: expand_aggregate(t, q, slide), prep={"slide": slide},
                  unselected=UNSELECTED)


# ---- the checks of one case --------------------------------------------------------------------------------------------
def _m2_col(res, j):
    return res.names[j][1] == "m2"


def _pair_moment(res, j):
    return res.names[j][1] in ("c", "m2x", "m2y")


def assert_identical(a, b, what, nan_equal=False, pair_moments=True):
    """Byte for byte (nan_equal: an M2 cell that is NaN in both matches whatever its payload; pair_moments=False leaves
    out the pairs' C, M2x and M2y)."""
    assert a.names == b.names
    assert (a.validity == b.validity).all(), "%s: validity differs" % what
    for j, name in enumerate(a.names):
        if not pair_moments and _pair_moment(a, j):
            continue
        x, y = a.values[j], b.values[j]
        same = x == y
        if nan_equal and _m2_col(a, j):
            same |= np.isnan(x.view(np.float64)) & np.isnan(y.view(np.float64))
        assert same.all(), "%s: %s differs at cells %s" % (what, name, np.nonzero(~same)[0][:5])


def _added_in_f64(res, j):
    col, agg = res.names[j]
    return agg in ("mean", "m2", "c", "m2x", "m2y") or (agg == "sum" and res.phys[col] == F64)


def assert_same_but_f64_sums(a, b, what):
    assert a.names == b.names and (a.validity == b.validity).all(), what
    for j, name in enumerate(a.names):
        if not _added_in_f64(a, j):
            assert (a.values[j] == b.values[j]).all(), "%s: %s differs" % (what, name)


def without_moments(res):
    """res without its M2 and pair outputs (assert_matches_exact compares every output it does not know bit for bit;
    check_m2 holds M2 to its tolerance, check_pair the pairs)."""
    keep = [j for j, (_, agg) in enumerate(res.names) if agg not in ("m2", "n", "c", "m2x", "m2y")]
    out = copy.copy(res)
    out.names = [res.names[j] for j in keep]
    out.values, out.validity = res.values[keep], res.validity[keep]
    if hasattr(res, "center"):
        out.center = {keep.index(j): v for j, v in res.center.items() if j in keep}
        out.bound = {keep.index(j): v for j, v in res.bound.items() if j in keep}
    return out


def check_int_mean_pin(got, exp, shard_exps, what):
    """Every integer MEAN cell equals rank_order_mean of the shards' exact sums in gather order, bit for bit."""
    for j, (col, agg) in enumerate(got.names):
        if agg != "mean" or exp.phys[col] == F64:
            continue
        cells = sorted(exp.exact_sums[col])
        want = np.array([rank_order_mean([se.exact_sums.get(col, {}).get(c, (0, 0))[0] for se in shard_exps],
                                         exp.exact_sums[col][c][1]) for c in cells], dtype=np.float64)
        g = got.values[j][cells]
        bad = np.nonzero(g != want.view(np.uint64))[0]
        assert bad.size == 0, "%s: col %s integer MEAN at cells %s: got %s, rank order gives %s" % (
            what, col, np.asarray(cells)[bad[:3]], g[bad[:3]].view(np.float64), want[bad[:3]])


def check_case(engine, fam, n, layout, shards, order):
    what = "%s N=%d %s" % (fam.name, n, layout)
    exp = fam.expected()
    with RankScans(engine, fam.arena, fam.descs, fam.q, shards, files=fam.files, tombstones=fam.tombstones,
                   **fam.prep) as rs:
        ctr = rs.run()
        assert len(set(rs.words())) == 1, "%s: exchange words %s" % (what, rs.words())
        whole = fam.whole_counters(engine)
        for k in COUNTERS:
            assert sum(c[k] for c in ctr) == whole[k], "%s: counter %s %s over ranks, %s whole" % (
                what, k, [c[k] for c in ctr], whole[k])
        plain = rs.finalize()[0] if n == 1 else None
        ranks = rs.gather(order)
        for r, res in enumerate(ranks[1:], 1):
            assert_identical(res, ranks[0], "%s: rank %d against rank 0" % (what, r))
        got = ranks[0]
        if fam.m2_rtol or fam.pair_rtol:
            if fam.m2_rtol:
                check_m2(got, exp, what, rtol=fam.m2_rtol)
            for k, ex in enumerate(fam.pairs() if fam.pair_rtol else []):
                check_pair(got, k, ex, rtol=fam.pair_rtol, what="%s pair %d" % (what, k))
            assert_matches_exact(without_moments(got), without_moments(exp), what=what, int_mean=False)
        else:
            assert_matches_exact(got, exp, what=what, int_mean=False)
        check_int_mean_pin(got, exp, [fam.shard_ref(shards[r]) for r in order], what)
        if plain is not None:
            assert_identical(got, plain, what + ": one rank against the plain finalize", nan_equal=True,
                             pair_moments=not fam.pair_rtol)
        if fam.m2_rtol or fam.pair_rtol:
            with pytest.raises(TskvError) as e:
                rs.scans[0].partials()
            assert e.value.status == cabi.TSKV_ERR_UNSUPPORTED
        else:
            for r, res in enumerate(rs.allreduce(order)):
                assert_identical(res, got, "%s: all-reduce on rank %d against the gather" % (what, r))
        if list(order) != sorted(order):
            assert_same_but_f64_sums(got, rs.gather()[0], what + ": reversed against forward order")
    return got


def run_family(engine, fam, n, monkeypatch, only=None):
    for k, v in fam.env.items():
        monkeypatch.setenv(k, v)
    cases = layouts(fam.all_ids, n, fam.unselected)
    for layout, (shards, order) in cases.items():
        if only is None or layout in only:
            check_case(engine, fam, n, layout, shards, order)
    return len(cases) if only is None else len(only)


@pytest.mark.parametrize("n", NS)
@pytest.mark.parametrize("name", FAMILIES)
def test_family(engine, name, n, monkeypatch):
    run_family(engine, family(name), n, monkeypatch)


# ---- M2 arenas ---------------------------------------------------------------------------------------------------------
def far_apart_values(rng, rank, n, kind):
    """Values of rank `rank`'s series: around rank * 1e6 ("steps"), or around +-1e12 by rank parity ("alternating")."""
    if kind == "steps":
        return rank * 1e6 + rng.normal(0, 1, n)
    return (1e12 if rank % 2 else -1e12) + rng.normal(0, 1, n)


def near_2_63_values(rng, rank, n, pt):
    """Exact in f64, every rank's mean near 2^63 in magnitude: u64 2^63 + 2048 k, i64 -2^63 + 1024 k, k spread by rank."""
    k = rank * 100_000 + rng.integers(0, 64, n)
    if pt == U64:
        return (np.uint64(2**63) + np.uint64(2048) * k.astype(np.uint64)).astype(np.uint64)
    return (np.int64(-2**63) + np.int64(1024) * k.astype(np.int64)).astype(np.int64)


def ill_conditioned_values(rng, n):
    return 1e9 + rng.normal(0, 1e-3, n)


def rank_arena(n_ranks, per_rank, rows, values, fields, first_half=()):
    """per_rank series for each of n_ranks ranks (series r * per_rank .. : rank r under the contiguous layout), rows
    rows each on the STEP grid (jittered below it); values(rng, rank, sid, n, pt) gives a series' column. Series of the ranks
    in first_half stop half way, so the later cells hold none of their values."""
    rng = np.random.default_rng(17)
    b = datagen.ArenaBuilder()
    truth = {}
    for r in range(n_ranks):
        for i in range(per_rank):
            sid = r * per_rank + i
            m = rows // 2 if r in first_half else rows
            ts = T0 + np.arange(m, dtype=np.int64) * STEP + rng.integers(0, STEP // 2, m)
            fl, cols = [], {}
            for col, pt in fields:
                v = values(rng, r, sid, m, pt)
                fl.append((col, pt, v, None))
                cols[col] = (v, np.ones(m, dtype=bool))
            b.add_column_group(sid, ts, fl)
            truth[sid] = [(ts, cols)]
    arena, descs = b.finish()
    return arena, descs, truth


def m2_family(name, arena, descs, truth, width, fields, rtol, gbs=False):
    q = QueryOption([PushedAggregate(c, pt, M2_AGGS) for c, pt in fields], series_ids=np.array(sorted(truth), np.uint32),
                    group_by_series=gbs, **_grid(truth, width))
    return Family(name, arena, descs, truth, q, _plain_ref(q), m2_rtol=rtol)


@pytest.mark.parametrize("kind,n,layout", [("steps", 8, "contiguous"), ("alternating", 4, "mod")])
def test_m2_far_apart_means(engine, kind, n, layout, monkeypatch):
    """The between-rank term n_r (mu_r - mu)^2 dominates M2."""
    fields = ((1, I64), (2, F64))

    def values(rng, r, sid, m, pt):  # alternating: the sign of series sid % 4 == rank under the mod layout
        x = far_apart_values(rng, r if kind == "steps" else sid % 2, m, kind)
        return np.round(x).astype(np.int64) if pt == I64 else x
    arena, descs, truth = rank_arena(8, 3, 120, values, fields)
    for gbs in (False, True):
        fam = m2_family("far apart %s gbs=%s" % (kind, gbs), arena, descs, truth, 30_000, fields, 1e-9, gbs)
        run_family(engine, fam, n, monkeypatch, only=(layout,))
        run_family(engine, fam, 1, monkeypatch)
        if not gbs:  # the cells do hold every rank's values, and the spread between ranks is what M2 holds
            exp = fam.expected()
            j = exp.names.index((2, "m2"))
            x = np.concatenate([truth[s][0][1][2][0] for s in truth])
            assert exp.validity[j].any() and exact_m2(x) > 1e6 * x.size


@pytest.mark.parametrize("gbs", [False, True])
def test_m2_means_near_2_63(engine, gbs, monkeypatch):
    """u64 2^63 + 2048 k and i64 -2^63 + 1024 k (exact in f64); rank 0's series stop half way, so the later cells take
    their shift from rank 1. By series, one rank holds each cell."""
    fields = ((1, I64), (3, U64))
    arena, descs, truth = rank_arena(4, 4, 200, lambda rng, r, sid, m, pt: near_2_63_values(rng, r, m, pt), fields,
                                     first_half=(0,))
    fam = m2_family("near 2^63 gbs=%s" % gbs, arena, descs, truth, 25_000, fields, 1e-9, gbs)
    run_family(engine, fam, 4, monkeypatch, only=("contiguous", "empty"))
    run_family(engine, fam, 1, monkeypatch)
    exp = fam.expected()
    j = exp.names.index((3, "count"))
    late = np.arange(exp.values.shape[1]) % fam.q.n_buckets >= fam.q.n_buckets * 3 // 4
    assert (exp.values[j][late & exp.validity[j]] > 0).any()  # later cells hold values, none from rank 0


def test_m2_ill_conditioned(engine, monkeypatch):
    """1e9 + N(0, 1e-3), one series per rank with 1-3 values of each cell."""
    arena, descs, truth = rank_arena(8, 1, 400, lambda rng, r, sid, m, pt: ill_conditioned_values(rng, m), ((2, F64),))
    fam = m2_family("ill-conditioned", arena, descs, truth, 2_500, ((2, F64),), 1e-6)
    run_family(engine, fam, 8, monkeypatch, only=("contiguous", "mod", "reversed"))
    run_family(engine, fam, 1, monkeypatch)


def special_arena():
    """One series per rank of 8, width W buckets: bucket 0 one value each, series 1's NaN; bucket 1 one value each, series
    2's +inf; bucket 2 one value of series 5 only; bucket 3 none; bucket 4 one value each (var_samp of 8 values)."""
    rng = np.random.default_rng(23)
    w = 10_000
    b = datagen.ArenaBuilder()
    truth = {}
    for sid in range(8):
        buckets = [0, 1] + ([2] if sid == 5 else []) + [4]
        ts = T0 + np.array(buckets, dtype=np.int64) * w + sid * 10
        f = rng.normal(0, 1e3, ts.size)
        if sid == 1:
            f[0] = math.nan
        if sid == 2:
            f[1] = math.inf
        i = rng.integers(-10**15, 10**15, ts.size)
        cols = {1: (i, np.ones(ts.size, dtype=bool)), 2: (f, np.ones(ts.size, dtype=bool))}
        b.add_column_group(sid, ts, [(1, I64, i, None), (2, F64, f, None)])
        truth[sid] = [(ts, cols)]
    arena, descs = b.finish()
    return arena, descs, truth, w


def test_m2_special_values_and_small_cells(engine, monkeypatch):
    arena, descs, truth, w = special_arena()
    fields = ((1, I64), (2, F64))
    q = QueryOption([PushedAggregate(c, pt, M2_AGGS + ("var_samp",)) for c, pt in fields],
                    series_ids=np.arange(8, dtype=np.uint32), width=w, first_bucket_start=T0, n_buckets=5)
    fam = Family("special", arena, descs, truth, q, _plain_ref(q), m2_rtol=1e-9)
    for n in (8, 1):
        got = None
        for layout, (shards, order) in layouts(fam.all_ids, n).items():
            if layout in ("contiguous", "reversed", "whole"):
                got = check_case(engine, fam, n, layout, shards, order)
        m2, ok = got.column(2, "m2")
        assert np.isnan(m2[0, 0]) and np.isnan(m2[0, 1]) and ok[0, 2] and m2[0, 2] == 0.0 and not ok[0, 3]
        m2, ok = got.column(1, "m2")
        assert ok[0, 2] and m2[0, 2] == 0.0 and not ok[0, 3]
        for col in (1, 2):
            v, ok = got.column(col, "var_samp")
            x = [float(truth[s][0][1][col][0][-1]) for s in range(8)]
            assert ok[0, 4] and abs(v[0, 4] - exact_m2(x) / 7) <= 1e-9 * exact_m2(x) / 7, (col, v[0, 4])


# ---- column pairs through k_merge_pairs on the M2 arenas -------------------------------------------------------------
def pair_family(name, arena, descs, truth, width, fields, pairs, rtol, gbs=False):
    q = QueryOption([PushedAggregate(c, pt, ("count",)) for c, pt in fields],
                    series_ids=np.array(sorted(truth), np.uint32), group_by_series=gbs, pairs=pairs,
                    **_grid(truth, width))
    return Family(name, arena, descs, truth, q, _plain_ref(q), pair_rtol=rtol)


@pytest.mark.parametrize("kind,n,layout", [("steps", 8, "contiguous"), ("alternating", 4, "mod")])
def test_pairs_far_apart_means(engine, kind, n, layout, monkeypatch):
    """The between-rank terms n_r (mx_r - mx)(my_r - my) dominate C, M2x and M2y."""
    fields = ((1, I64), (2, F64))

    def values(rng, r, sid, m, pt):
        x = far_apart_values(rng, r if kind == "steps" else sid % 2, m, kind)
        return np.round(x).astype(np.int64) if pt == I64 else x
    arena, descs, truth = rank_arena(8, 3, 120, values, fields)
    pairs = [(1, I64, 2, F64), (2, F64, 2, F64), (2, F64, 1, I64)]
    for gbs in (False, True):
        fam = pair_family("pairs far apart %s gbs=%s" % (kind, gbs), arena, descs, truth, 30_000, fields, pairs, 1e-9,
                          gbs)
        run_family(engine, fam, n, monkeypatch, only=(layout,))
        run_family(engine, fam, 1, monkeypatch)
        if not gbs:  # the spread between ranks is what C holds
            n_e, c_e, _, _ = fam.pairs()[0]
            assert (n_e > 0).any() and np.abs(c_e[n_e > 0]).max() > 1e12


@pytest.mark.parametrize("gbs", [False, True])
def test_pairs_means_near_2_63(engine, gbs, monkeypatch):
    """u64 2^63 + 2048 k against i64 -2^63 + 1024 k (exact in f64); rank 0's series stop half way, so the later cells
    take their shifts from rank 1 (and, with the "empty" layout, rank 0 holds no page)."""
    fields = ((1, I64), (3, U64))
    arena, descs, truth = rank_arena(4, 4, 200, lambda rng, r, sid, m, pt: near_2_63_values(rng, r, m, pt), fields,
                                     first_half=(0,))
    pairs = [(1, I64, 3, U64), (3, U64, 3, U64), (1, I64, 1, I64)]
    fam = pair_family("pairs near 2^63 gbs=%s" % gbs, arena, descs, truth, 25_000, fields, pairs, 1e-9, gbs)
    run_family(engine, fam, 4, monkeypatch, only=("contiguous", "empty"))
    run_family(engine, fam, 1, monkeypatch)
    n_e = fam.pairs()[0][0]
    late = np.arange(n_e.size) % fam.q.n_buckets >= fam.q.n_buckets * 3 // 4
    assert (n_e[late] > 0).any()  # later cells hold pairs, none from rank 0


def test_pairs_ill_conditioned(engine, monkeypatch):
    """1e9 + N(0, 1e-3) in both operands, one series per rank with 1-3 rows of each cell."""
    fields = ((2, F64), (4, F64))
    arena, descs, truth = rank_arena(8, 1, 400, lambda rng, r, sid, m, pt: ill_conditioned_values(rng, m), fields)
    fam = pair_family("pairs ill-conditioned", arena, descs, truth, 2_500, fields, [(2, F64, 4, F64), (4, F64, 4, F64)],
                      1e-6)
    run_family(engine, fam, 8, monkeypatch, only=("contiguous", "mod", "reversed"))
    run_family(engine, fam, 1, monkeypatch)

