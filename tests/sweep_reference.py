"""Cases for the kernel sweep (tests/test_gpu_kernel_sweep.py), with no GPU code: arenas aimed at any bin of the fused scan,
random combinations of query features, page-set options and scan switches, and the composed exact reference of each.

The fused scan runs one kernel instantiation per (decode-kind bin, FIRST / LAST, narrow flag, edge scan), and the M2
second pass one per (bin, edge scan): INSTANTIATIONS lists them all by hand, and tests/test_kernel_list.py holds that list
to the kernels the built library contains. A bin is a time codec (RLE, simple8b, or generic: raw / NULL time pages) x a
value codec (simple8b, Gorilla, or generic: raw, run-length, boolean, all-NULL); bins 9-12 hold the simple8b / Gorilla
value pages of at most SHORT_PAGE_ROWS rows behind RLE / simple8b time pages and run the kernels of their serial bin.
kernel_keys reads back which instantiations a pass ran on field pages from its work list (PreparedScan.work_list()).

A case's expected outcome is the exact reference of tests/helpers.py composed for its features (edges, labels, GROUP BY
tags, sliding windows, M2, tombstones, the overlap merge), or the status the scan must refuse it with: the reference's own
ReferenceError, or a refusal this module states: SUM or M2 on a BOOL column (TSKV_ERR_INVALID_ARG), FIRST / LAST with a
sliding window (TSKV_ERR_UNSUPPORTED, sliding_reference.sliding_status), M2 with a sliding window (the engine's
ValueError, before the library is called).

random_operand_case adds column pairs (covar / corr) and medians to a random case. Their outcome adds the exact
co-moments (covariance_reference) and medians (median_reference) of every pair and median, or one more refusal this
module states: a pair or a median with a sliding window (the engine's ValueError), a BOOL operand
(TSKV_ERR_INVALID_ARG). The scan runs such a query with every operand that is not projected as a COUNT column without
output (scan_query): the other outputs' reference is that query's.

random_increase_case adds counter increases (increase(time, x)) to a random case, and regroups most cases into a shape
whose cells hold one series. Their outcome adds the exact increase of every increase (increase_reference), or the
status of increase_status: the refusals of validate_query (cnosdb_b200/csrc/tskv_gpu.cu) in the order it checks them."""
import copy

import numpy as np

from cnosdb_b200 import cabi, datagen
from cnosdb_b200.engine import PushedAggregate, QueryOption, sliding_window_grid
from tests.edges_reference import exact_aggregate_edges, exact_aggregate_grouped_edges
from tests.exact_arenas import add_column_group, merge_truth
from tests.group_reference import exact_aggregate_grouped
from tests.helpers import ReferenceError, bucket_spec, exact_aggregate, files_by_series, overlap_groups
from tests.labels_reference import exact_aggregate_grouped_labels, exact_aggregate_labels
from tests.sliding_reference import expand_aggregate, sliding_status
from tests.covariance_reference import exact_pair_cells
from tests.increase_reference import exact_increase_cells
from tests.median_reference import exact_median_cells
from tests.variance_reference import with_m2

# ---- the kernels -------------------------------------------------------------------------------------------------------
TK_RLE, TK_S8B, TK_GEN = 0, 1, 2
VK_S8B, VK_GOR, VK_GEN = 0, 1, 2
N_VK = 3
NARROW_NONE, NARROW_SOME, NARROW_ALL = 0, 1, 2
N_SERIAL_BINS, N_BINS = 9, 13
SHORT_PAGE_ROWS = 1024
# short-page bin -> the serial bin whose kernels run it (RLE / simple8b time x simple8b / Gorilla values)
SHORT_BINS = {9: TK_RLE * N_VK + VK_S8B, 10: TK_S8B * N_VK + VK_S8B, 11: TK_RLE * N_VK + VK_GOR, 12: TK_S8B * N_VK + VK_GOR}
SCAN, M2 = "k_scan_aggregate", "k_scan_m2"

# (kernel, TK, VK, SEL, NARROW, EDGES). k_scan_m2 has no FIRST / LAST or narrow variants: SEL False, NARROW_NONE.
INSTANTIATIONS = [
    # pass 1 without FIRST / LAST: every bin, and the narrow variants of the simple8b-value bins behind RLE / simple8b time
    (SCAN, TK_RLE, VK_S8B, False, NARROW_NONE, False), (SCAN, TK_RLE, VK_S8B, False, NARROW_NONE, True),
    (SCAN, TK_RLE, VK_S8B, False, NARROW_SOME, False), (SCAN, TK_RLE, VK_S8B, False, NARROW_SOME, True),
    (SCAN, TK_RLE, VK_S8B, False, NARROW_ALL, False), (SCAN, TK_RLE, VK_S8B, False, NARROW_ALL, True),
    (SCAN, TK_RLE, VK_GOR, False, NARROW_NONE, False), (SCAN, TK_RLE, VK_GOR, False, NARROW_NONE, True),
    (SCAN, TK_RLE, VK_GEN, False, NARROW_NONE, False), (SCAN, TK_RLE, VK_GEN, False, NARROW_NONE, True),
    (SCAN, TK_S8B, VK_S8B, False, NARROW_NONE, False), (SCAN, TK_S8B, VK_S8B, False, NARROW_NONE, True),
    (SCAN, TK_S8B, VK_S8B, False, NARROW_SOME, False), (SCAN, TK_S8B, VK_S8B, False, NARROW_SOME, True),
    (SCAN, TK_S8B, VK_S8B, False, NARROW_ALL, False), (SCAN, TK_S8B, VK_S8B, False, NARROW_ALL, True),
    (SCAN, TK_S8B, VK_GOR, False, NARROW_NONE, False), (SCAN, TK_S8B, VK_GOR, False, NARROW_NONE, True),
    (SCAN, TK_S8B, VK_GEN, False, NARROW_NONE, False), (SCAN, TK_S8B, VK_GEN, False, NARROW_NONE, True),
    (SCAN, TK_GEN, VK_S8B, False, NARROW_NONE, False), (SCAN, TK_GEN, VK_S8B, False, NARROW_NONE, True),
    (SCAN, TK_GEN, VK_GOR, False, NARROW_NONE, False), (SCAN, TK_GEN, VK_GOR, False, NARROW_NONE, True),
    (SCAN, TK_GEN, VK_GEN, False, NARROW_NONE, False), (SCAN, TK_GEN, VK_GEN, False, NARROW_NONE, True),
    # pass 1 with FIRST / LAST: every bin
    (SCAN, TK_RLE, VK_S8B, True, NARROW_NONE, False), (SCAN, TK_RLE, VK_S8B, True, NARROW_NONE, True),
    (SCAN, TK_RLE, VK_GOR, True, NARROW_NONE, False), (SCAN, TK_RLE, VK_GOR, True, NARROW_NONE, True),
    (SCAN, TK_RLE, VK_GEN, True, NARROW_NONE, False), (SCAN, TK_RLE, VK_GEN, True, NARROW_NONE, True),
    (SCAN, TK_S8B, VK_S8B, True, NARROW_NONE, False), (SCAN, TK_S8B, VK_S8B, True, NARROW_NONE, True),
    (SCAN, TK_S8B, VK_GOR, True, NARROW_NONE, False), (SCAN, TK_S8B, VK_GOR, True, NARROW_NONE, True),
    (SCAN, TK_S8B, VK_GEN, True, NARROW_NONE, False), (SCAN, TK_S8B, VK_GEN, True, NARROW_NONE, True),
    (SCAN, TK_GEN, VK_S8B, True, NARROW_NONE, False), (SCAN, TK_GEN, VK_S8B, True, NARROW_NONE, True),
    (SCAN, TK_GEN, VK_GOR, True, NARROW_NONE, False), (SCAN, TK_GEN, VK_GOR, True, NARROW_NONE, True),
    (SCAN, TK_GEN, VK_GEN, True, NARROW_NONE, False), (SCAN, TK_GEN, VK_GEN, True, NARROW_NONE, True),
    # pass 2 of M2: every bin
    (M2, TK_RLE, VK_S8B, False, NARROW_NONE, False), (M2, TK_RLE, VK_S8B, False, NARROW_NONE, True),
    (M2, TK_RLE, VK_GOR, False, NARROW_NONE, False), (M2, TK_RLE, VK_GOR, False, NARROW_NONE, True),
    (M2, TK_RLE, VK_GEN, False, NARROW_NONE, False), (M2, TK_RLE, VK_GEN, False, NARROW_NONE, True),
    (M2, TK_S8B, VK_S8B, False, NARROW_NONE, False), (M2, TK_S8B, VK_S8B, False, NARROW_NONE, True),
    (M2, TK_S8B, VK_GOR, False, NARROW_NONE, False), (M2, TK_S8B, VK_GOR, False, NARROW_NONE, True),
    (M2, TK_S8B, VK_GEN, False, NARROW_NONE, False), (M2, TK_S8B, VK_GEN, False, NARROW_NONE, True),
    (M2, TK_GEN, VK_S8B, False, NARROW_NONE, False), (M2, TK_GEN, VK_S8B, False, NARROW_NONE, True),
    (M2, TK_GEN, VK_GOR, False, NARROW_NONE, False), (M2, TK_GEN, VK_GOR, False, NARROW_NONE, True),
    (M2, TK_GEN, VK_GEN, False, NARROW_NONE, False), (M2, TK_GEN, VK_GEN, False, NARROW_NONE, True),
]


def serial_bin(b):
    return SHORT_BINS.get(b, b)


def key_name(key):
    kernel, tk, vk, sel, narrow, edges = key
    name = lambda names, k: names[k] if 0 <= k < len(names) else str(k)  # noqa: E731  (a kernel the list does not know)
    return "%s<%s, %s, %s, %s, %s>" % (kernel, name(("TK_RLE", "TK_S8B", "TK_GEN"), tk),
                                       name(("VK_S8B", "VK_GOR", "VK_GEN"), vk), sel,
                                       name(("NARROW_NONE", "NARROW_SOME", "NARROW_ALL"), narrow), edges)


def bin_narrow_flags(wl, descs):
    """NARROW_* of every bin: over all field pages of the page set, none, some or all narrow."""
    field = descs["phys_type"] != cabi.TSKV_PT_TIME
    out = []
    for b in range(N_BINS):
        m = field & (wl["page_bin"] == b)
        n, k = int(m.sum()), int(wl["page_narrow"][m].astype(bool).sum())
        out.append(NARROW_NONE if k == 0 else NARROW_ALL if k == n else NARROW_SOME)
    return out


def bin_fill(wl, n_cols):
    """Work-list items of every (bin, query column): the fills of its narrow and wide buckets."""
    return wl["fill"].astype(np.int64).reshape(N_BINS, n_cols, 2).sum(axis=2)


def kernel_keys(wl, descs, query, edges):
    """-> ({instantiation key: bins}, ...) of the kernels a pass ran on field pages: every bin whose work list holds items
    runs scan_kernel_for(serial bin, FIRST / LAST, narrow flag, edges), and M2 columns' items run k_scan_m2 once more."""
    has_sel = any(c.agg_mask & (cabi.TSKV_AGG_FIRST | cabi.TSKV_AGG_LAST) for c in query.columns)
    m2_cols = [j for j, c in enumerate(query.columns) if c.agg_mask & cabi.TSKV_AGG_M2]
    fill = bin_fill(wl, len(query.columns))
    narrow = bin_narrow_flags(wl, descs)
    out = {}
    for b in range(N_BINS):
        if not fill[b].sum():
            continue
        sb = serial_bin(b)
        tk, vk = divmod(sb, N_VK)
        nf = narrow[b] if (not has_sel and tk != TK_GEN and vk == VK_S8B) else NARROW_NONE
        out.setdefault((SCAN, tk, vk, has_sel, nf, bool(edges)), set()).add(b)
        if m2_cols and fill[b, m2_cols].sum():
            out.setdefault((M2, tk, vk, False, NARROW_NONE, bool(edges)), set()).add(b)
    return out


# ---- values and column groups ------------------------------------------------------------------------------------------
T0 = 10**12
I64, F64, U64, BOOL = cabi.TSKV_PT_I64, cabi.TSKV_PT_F64, cabi.TSKV_PT_U64, cabi.TSKV_PT_BOOL
COLUMNS = {1: I64, 2: F64, 3: U64, 4: BOOL}
# value encodings by physical type: simple8b narrow / wide (values inside / outside the 32-bit range), run-length (an
# arithmetic sequence), raw (Encoding::Null), Gorilla, bit-packed / one-byte booleans
ENCODINGS = {I64: ("s8b_narrow", "s8b_wide", "rle", "raw"), U64: ("s8b_narrow", "s8b_wide", "raw"),
             F64: ("gorilla", "raw"), BOOL: ("pack", "raw")}


def column_values(rng, pt, enc, n):
    """Values of one page. Wide integers stay exact in f64 (M2 converts them), u64 ones lie above 2^63."""
    walk = np.cumsum(rng.integers(-3, 4, n))
    walk[n // 2:] += 5 * (n >= 3)  # (equal deltas, the abs() below included, would make a run-length page)
    if pt == BOOL:
        return rng.random(n) < 0.5
    if pt == F64:
        return walk.astype(np.float64) + np.round(rng.random(n), 3)
    if enc == "rle":
        return (int(rng.integers(-1000, 1000)) + np.arange(n) * int(rng.integers(1, 9))).astype(np.int64)
    if pt == U64:
        if enc == "s8b_narrow":
            return (np.abs(walk) + int(rng.integers(0, 2**31 - 10**4))).astype(np.uint64)
        return np.uint64(2**63) + (np.abs(walk) * 2048).astype(np.uint64)  # multiples of 2^11: exact as f64
    if enc == "s8b_narrow":
        return (walk + int(rng.integers(-2**31 + 10**4, 2**31 - 10**4))).astype(np.int64)
    return (walk + int(rng.choice([-1, 1])) * 2**40).astype(np.int64)


def encoder(pt, enc):
    if enc == "raw":
        return datagen.encode_bools_raw if pt == BOOL else datagen.encode_raw
    return None  # ArenaBuilder's default: simple8b / run-length integers, Gorilla floats, bit-packed booleans


def timestamps(rng, kind, t_start, n, step):
    """RLE: a regular grid; s8b: jittered below the step (strictly increasing); raw: either, behind a raw time page."""
    k = np.arange(n, dtype=np.int64)
    ts = t_start + k * step
    if kind == "s8b" or (kind == "raw" and rng.random() < 0.5):
        if step >= 2 and n > 1:
            jit = rng.integers(0, step, n)
            jit[0] = 0
            if n >= 3 and np.unique(np.diff(jit)).size == 1:
                jit[1] = (jit[1] + 1) % step  # (equal deltas would make a run-length time page)
            ts = ts + jit
    return ts


class Arena:
    """ArenaBuilder + the truth of the exact references ({sid: [(ts, {col: (values, valid)})]})."""

    def __init__(self):
        self.b = datagen.ArenaBuilder()
        self.truth = {}

    def add(self, rng, sid, ts, time_kind, cols, null_frac):
        """cols: [(column id, encoding)]. null_frac 1.0: all-NULL pages."""
        n = len(ts)
        fl, tc = [], {}
        for col, enc in cols:
            pt = COLUMNS[col]
            vals = column_values(rng, pt, enc, n)
            valid = rng.random(n) >= null_frac if null_frac else np.ones(n, dtype=bool)
            if enc == "rle" and not valid.all():
                valid[:] = True  # (a NULL would break the arithmetic sequence of the kept values)
            fl.append((col, pt, vals, None if valid.all() else valid, encoder(pt, enc)))
            tc[col] = (vals, valid)
        add_column_group(self.b, sid, ts, fl, raw_time=time_kind == "raw")
        self.truth.setdefault(sid, []).append((np.asarray(ts, dtype=np.int64), tc))

    def finish(self):
        arena, descs = self.b.finish()
        return arena, descs, self.truth


# ---- arenas aimed at one bin -------------------------------------------------------------------------------------------
BIN_STEP = 1000
HELPER_SERIES = (1000, 1001)


def bin_arena(b, narrow=NARROW_NONE, seed=0):
    """Every field page in bin b. Simple8b values: NARROW_NONE wide pages only, NARROW_ALL narrow ones only, NARROW_SOME
    33 wide and 31 narrow pages per column, so that the wide bucket ends in a chunk of one page (the other 31 lanes of the
    chunk's narrow vote hold no page). The simple8b-value bins behind RLE / simple8b time also get HELPER_SERIES. Long
    bins (0-8 with simple8b / Gorilla values behind RLE / simple8b time) take pages of 1025-1500 rows, short bins 8-1024;
    the generic-value bins hold raw, run-length, boolean and all-NULL pages."""
    rng = np.random.default_rng([b, narrow, seed])
    sb = serial_bin(b)
    tk, vk = divmod(sb, N_VK)
    time_kind = ("rle", "s8b", "raw")[tk]
    a = Arena()
    n_series = 64 if narrow == NARROW_SOME else 40
    for sid in range(n_series):
        if b >= N_SERIAL_BINS:  # (the writer may store pages of a few rows in another codec)
            n = int(rng.choice([8, 31, 32, 33, int(rng.integers(34, SHORT_PAGE_ROWS + 1)), SHORT_PAGE_ROWS]))
        elif vk != VK_GEN and tk != TK_GEN:
            n = int(rng.integers(SHORT_PAGE_ROWS + 1, 1501))
        else:
            n = int(rng.choice([1 if tk == TK_GEN == vk else 8, 33, int(rng.integers(34, 1501))]))
        ts = timestamps(rng, time_kind, T0 + (sid % 7) * BIN_STEP, n, BIN_STEP)
        null_frac = 0.2 if sid % 3 == 1 else 0.0
        if vk == VK_S8B:
            wide = narrow == NARROW_NONE or (narrow == NARROW_SOME and sid < 33)
            enc = "s8b_wide" if wide else "s8b_narrow"
            cols = [(1, enc), (3, enc)]
        elif vk == VK_GOR:
            cols = [(2, "gorilla")]
        else:
            # (a run-length page of one or two values would be written as simple8b)
            cols = [(1, "rle" if sid % 4 == 0 and n >= 3 else "raw"), (2, "raw"), (3, "raw"), (4, ("pack", "raw")[sid % 2])]
            if sid % 9 == 5:
                null_frac = 1.0
        a.add(rng, sid, ts, time_kind, cols, null_frac)
    if sb in (TK_RLE * N_VK + VK_S8B, TK_S8B * N_VK + VK_S8B):
        # HELPER_SERIES: a narrow and a wide page in a short bin of the other time codec (so that bin is NARROW_SOME). The
        # scan then keeps narrow pages apart and its work list reports every page's narrow flag; targeted_query leaves
        # these series out, so their bin runs no item.
        other = "s8b" if tk == TK_RLE else "rle"
        for sid, enc in zip(HELPER_SERIES, ("s8b_narrow", "s8b_wide")):
            a.add(rng, sid, timestamps(rng, other, T0, 100, BIN_STEP), other, [(1, enc), (3, enc)], 0.0)
    return a.finish()


# ---- queries -----------------------------------------------------------------------------------------------------------
PLAIN = ("count", "sum", "min", "max", "mean")
SEL = ("count", "sum", "min", "max", "mean", "first", "last")
M2_AGGS = ("count", "min", "max", "mean", "m2")
BOOL_AGGS = {"plain": ("count", "min", "max"), "sel": ("count", "min", "max", "first", "last"), "m2": ("count", "max")}


def span(truth):
    ts = np.concatenate([t for cgs in truth.values() for t, _ in cgs])
    return int(ts.min()), int(ts.max())


def random_edges(rng, lo, hi, n):
    """n + 1 or fewer increasing edges over [lo, hi + 1], some 1 apart (buckets narrower than a time step)."""
    cuts = rng.integers(lo + 1, hi + 1, max(n - 1, 0))
    cuts = np.concatenate([cuts, cuts[: n // 5] + 1])
    return np.unique(np.concatenate([[lo], cuts, [hi + 1]])).astype(np.int64)


def columns_of(truth):
    return sorted({c for cgs in truth.values() for _, cols in cgs for c in cols})


def kind_columns(truth, kind):
    """Every column of the arena with the aggregates of `kind` ("plain", "sel" with FIRST / LAST, "m2")."""
    aggs = {"plain": PLAIN, "sel": SEL, "m2": M2_AGGS}[kind]
    return [PushedAggregate(c, COLUMNS[c], BOOL_AGGS[kind] if COLUMNS[c] == BOOL else aggs) for c in columns_of(truth)]


def targeted_query(truth, key, seed=0):
    """The query of the targeted case of `key`: its aggregates, and an edge scan or a tumbling one."""
    kernel, _, _, sel, _, edges = key
    cols = kind_columns(truth, "m2" if kernel == M2 else "sel" if sel else "plain")
    ids = np.array([s for s in sorted(truth) if s not in HELPER_SERIES], dtype=np.uint32)
    lo, hi = span({s: truth[s] for s in ids})
    if edges:
        e = random_edges(np.random.default_rng(seed), lo, hi, 40)
        return QueryOption(cols, series_ids=ids, n_buckets=e.size - 1), {"edges": e}
    w = 37 * BIN_STEP
    fbs, nb = bucket_spec(lo, hi, w)
    return QueryOption(cols, series_ids=ids, width=w, first_bucket_start=fbs, n_buckets=nb), {}


# ---- random cases ------------------------------------------------------------------------------------------------------
GROUPINGS = ("bucket", "series", "tags", "edges", "labels", "sliding", "unbucketed")
ENV_PARTS = (None, "1", "3")
ENV_SMEM = (None, "0")
MAX_ROWS = 64 * 1500


class Case:
    """One random case: arena, descs, truth, files, tombstones, page-set options (host_resident, verify_on_read), query,
    extra (the scan's slide, group_ids / n_groups, edges, labels), env (TSKV_PARTS, TSKV_SMEM_TABLE_KB; None: unset) and the
    description of every draw."""

    def __init__(self, index):
        self.index = index
        self.desc = {}

    def describe(self):
        return "case %d: %s" % (self.index, ", ".join("%s=%s" % kv for kv in self.desc.items()))


def _random_arena(rng, case):
    step = int(rng.choice([1000, 7, 10**6]))
    n_series = int(rng.integers(1, 65))
    use_files = rng.random() < 0.25
    mix = rng.random() < 0.5  # several column sets per series
    col_pool = [c for c in COLUMNS if rng.random() < 0.7] or [1]
    a = Arena()
    files = []
    budget = MAX_ROWS // n_series
    for sid in range(n_series):
        n_cg = int(rng.choice([1, 1, 2, 3]))
        t = T0 + int(rng.integers(0, 20)) * step
        fids = rng.permutation(n_cg) + 1
        for g in range(n_cg):
            r = rng.random()
            n = int(rng.integers(1, 34) if r < 0.2 else rng.integers(34, 1025) if r < 0.7 else rng.integers(1025, 1501))
            n = max(1, min(n, budget // n_cg))
            time_kind = str(rng.choice(["rle", "s8b", "raw"]))
            ts = timestamps(rng, time_kind, t, n, step)
            if use_files and rng.random() < 0.5:
                t = int(ts[0]) + int(rng.integers(0, max(n, 1))) * step  # the next chunk overlaps this one
            else:
                t = int(ts[-1]) + step * int(rng.integers(1, 4))
            cols = col_pool if not mix else ([c for c in col_pool if rng.random() < 0.7] or col_pool[:1])
            encs = [(c, str(rng.choice(ENCODINGS[COLUMNS[c]]))) for c in cols]
            nf = float(rng.choice([0.0, 0.0, 0.1, 0.5, 1.0], p=[0.4, 0.2, 0.2, 0.15, 0.05]))
            a.add(rng, sid, ts, time_kind, encs, nf)
            files.append(int(fids[g]))
    case.arena, case.descs, case.truth = a.finish()
    case.files = np.array(files, dtype=np.uint64) if use_files else None
    case.desc.update(series=n_series, step=step, column_groups=len(files), files=use_files,
                     columns=col_pool, rows=int(sum(len(t) for cgs in case.truth.values() for t, _ in cgs)))
    return step


def _random_tombstones(rng, truth, lo, hi):
    """Row drops of one series, column masks, and a page-set-wide row drop, over random sub-ranges."""
    out = []
    sids = sorted(truth)
    for _ in range(int(rng.integers(1, 12))):
        a = int(rng.integers(lo, hi + 1))
        b = a + int(rng.integers(0, max((hi - lo) // 5, 1)))
        sid = int(rng.choice(sids))
        r = rng.random()
        if r < 0.5:
            out.append((sid, int(rng.choice(list(COLUMNS))), a, b))
        elif r < 0.9:
            out.append((sid, None, a, b))
        else:
            out.append((None, None, a, a + (b - a) // 8))
    return cabi.tombstones(out)


def _predicate(rng, truth, col):
    """A comparison of column `col` against one of its values (+-1), or a constant outside them."""
    pt = COLUMNS[col]
    vals = [v[ok] for cgs in truth.values() for _, cols in cgs if col in cols for v, ok in [cols[col]]]
    vals = np.concatenate(vals) if vals else np.zeros(0)
    op = str(rng.choice(["==", "!=", "<", "<=", ">", ">="]))
    if vals.size == 0 or rng.random() < 0.1:
        c = {I64: -2**62, U64: 2**63 - 1, F64: -1e300}[pt]
    else:
        c = vals[int(rng.integers(0, vals.size))]
        c = float(c) if pt == F64 else int(c) + int(rng.integers(-1, 2))
        if pt == U64:
            c = min(max(c, 0), 2**64 - 1)
    return (col, pt, op, c)


def random_case(index, base_seed):
    """The index-th case of the sweep of `base_seed`."""
    rng = np.random.default_rng([base_seed, index])
    case = Case(index)
    step = _random_arena(rng, case)
    truth = case.truth
    lo, hi = span(truth)
    grouping = str(rng.choice(GROUPINGS))
    # aggregates: FIRST / LAST and M2 on some cases; at most one deliberate refusal
    refusal = str(rng.choice(["none", "bool_sum", "bool_m2", "sel_sliding", "m2_sliding"],
                             p=[0.9, 0.025, 0.025, 0.025, 0.025]))
    have = columns_of(truth)
    if refusal in ("bool_sum", "bool_m2") and BOOL not in [COLUMNS[c] for c in have]:
        refusal = "none"
    if refusal in ("sel_sliding", "m2_sliding"):
        grouping = "sliding"
    want_sel = refusal == "sel_sliding" or \
        (refusal == "none" and grouping not in ("sliding", "labels") and rng.random() < 0.4)
    want_m2 = refusal in ("m2_sliding", "bool_m2") or (refusal == "none" and grouping != "sliding" and rng.random() < 0.3)
    qcols = [c for c in have if rng.random() < 0.75] or have[:1]
    if refusal in ("bool_sum", "bool_m2"):
        qcols = sorted(set(qcols) | {c for c in have if COLUMNS[c] == BOOL})
    cols = []
    for c in qcols:
        pt = COLUMNS[c]
        pool = ["count", "min", "max"] + ([] if pt == BOOL else ["sum", "mean"])
        if want_sel:
            pool += ["first", "last"]
        aggs = [x for x in pool if rng.random() < 0.6] or ["count"]
        if want_m2 and (pt != BOOL or refusal == "bool_m2"):
            aggs.append("m2")
        if refusal == "bool_sum" and pt == BOOL:
            aggs.append("sum")
        cols.append(PushedAggregate(c, pt, aggs))
    # series selection, predicates, time ranges
    sids = sorted(truth)
    series_ids = None
    if len(sids) > 1 and rng.random() < 0.3:
        series_ids = np.array(sorted(rng.choice(sids, int(rng.integers(1, len(sids) + 1)), replace=False)), dtype=np.uint32)
    num = [c for c in qcols if COLUMNS[c] != BOOL]
    n_pred = int(rng.choice([0, 0, 1, 2])) if num else 0
    preds = [_predicate(rng, truth, int(rng.choice(num))) for _ in range(n_pred)]
    n_ranges = int(rng.choice([0, 0, 1, 2]))
    ranges = []
    for _ in range(n_ranges):
        a = int(rng.integers(lo - 2 * step, hi + 1))
        ranges.append((a, a + int(rng.integers(0, max(hi - lo, 1) + 1))))
    # grouping
    extra, kw = {}, {}
    if grouping in ("bucket", "series", "tags"):
        w = int(rng.choice([37, 100, 1000])) * step
        origin = int(rng.integers(-w, w))
        fbs, nb = bucket_spec(lo, hi, w, origin)
        kw = dict(width=w, origin=origin, first_bucket_start=fbs, n_buckets=nb, group_by_series=grouping == "series")
    elif grouping in ("edges", "labels"):
        e = random_edges(rng, lo, hi, int(rng.integers(1, 60)))
        extra["edges"] = e
        n_out = e.size - 1
        if grouping == "labels":
            n_out = int(rng.integers(1, 13))
            extra["labels"] = rng.integers(0, n_out, e.size - 1).astype(np.uint32)
        kw = dict(n_buckets=n_out, group_by_series=grouping == "edges" and rng.random() < 0.3)
    elif grouping == "sliding":
        slide = int(rng.choice([20, 50, 300])) * step
        window = slide * int(rng.integers(1, 5)) + (int(rng.integers(1, slide)) if rng.random() < 0.3 else 0)
        window += slide if window == slide else 0  # (slide == width is a tumbling scan)
        fbs, nb = sliding_window_grid(lo, hi, window, slide)
        kw = dict(width=window, first_bucket_start=fbs, n_buckets=nb, group_by_series=rng.random() < 0.3)
        extra["slide"] = slide
    else:
        kw = dict(group_by_series=rng.random() < 0.3)
    n_slots = len(series_ids) if series_ids is not None else len(sids)
    if grouping in ("tags", "labels", "edges") and not kw.get("group_by_series") and \
            (grouping == "tags" or rng.random() < 0.3):
        extra["n_groups"] = int(rng.integers(1, 6))
        extra["group_ids"] = rng.integers(0, extra["n_groups"], n_slots).astype(np.uint32)
    if grouping == "sliding" and case.files is not None:
        preds = []  # (the merged truth of the sliding reference holds no predicates)
    case.query = QueryOption(cols, series_ids=series_ids, time_ranges=ranges, predicates=preds, **kw)
    case.extra = extra
    # tombstones (not with sliding windows: their reference takes none), page-set options, scan switches
    case.tombstones = None
    if grouping != "sliding" and rng.random() < 0.3:
        case.tombstones = _random_tombstones(rng, truth, lo, hi)
    case.host_resident = bool(rng.random() < 0.25)
    case.verify_on_read = bool(rng.random() < 0.2)
    case.env = {"TSKV_PARTS": ENV_PARTS[int(rng.integers(0, 3))], "TSKV_SMEM_TABLE_KB": ENV_SMEM[int(rng.integers(0, 2))]}
    case.desc.update(grouping=grouping, refusal=refusal,
                     aggs={c.column_id: [cabi.AGG_NAMES[a] for a in c.agg_list()] for c in cols},
                     series_ids=None if series_ids is None else series_ids.tolist(), predicates=preds, ranges=ranges,
                     width=case.query.width, origin=case.query.origin, n_buckets=case.query.n_buckets,
                     group_by_series=case.query.group_by_series, slide=extra.get("slide"),
                     n_edges=None if "edges" not in extra else int(extra["edges"].size), n_groups=extra.get("n_groups"),
                     tombstones=0 if case.tombstones is None else len(case.tombstones),
                     host_resident=case.host_resident, verify_on_read=case.verify_on_read, env=case.env)
    return case


def expected(truth, query, extra, tombstones=None, files=None):
    """The composed exact reference of one scan -> ExactResult (M2 filled in; with pairs, medians or increases, `pairs`
    holds exact_pair_cells of every pair, `medians` exact_median_cells of every median and `increases`
    exact_increase_cells of every increase), or the status int the scan must refuse it with, or "ValueError" (the
    engine refuses M2, pairs, medians and increases with a sliding window before calling the library)."""
    medians = [c for c in query.columns if c.median]
    incs = [c for c in query.columns if c.increase]
    if query.pairs or medians or incs:
        if extra.get("slide") is not None:
            return "ValueError"
        if BOOL in [pt for _, pt in operands(query)]:
            return cabi.TSKV_ERR_INVALID_ARG
        st = increase_status(truth, query, extra) if incs else None
        if st is not None:
            return st
        res = expected(truth, scan_query(query), extra, tombstones, files)
        if isinstance(res, (int, str)):
            return res
        kw = dict(tombstones=tombstones, files=files, group_ids=extra.get("group_ids"), edges=extra.get("edges"),
                  labels=extra.get("labels"))
        n_cells = res.values.shape[1]
        res.pairs = [exact_pair_cells(truth, query, p, n_cells, **kw) for p in query.pairs]
        res.medians = [exact_median_cells(truth, query, c.column_id, c.phys_type, n_cells, **kw) for c in medians]
        kw.pop("labels")  # (labels refuse increases)
        res.increases = [exact_increase_cells(truth, query, c.column_id, c.phys_type, n_cells, **kw) for c in incs]
        return res
    has_m2 = any(c.agg_mask & cabi.TSKV_AGG_M2 for c in query.columns)
    has_sel = any(c.agg_mask & (cabi.TSKV_AGG_FIRST | cabi.TSKV_AGG_LAST) for c in query.columns)
    slide = extra.get("slide")
    if slide is not None and has_m2:
        return "ValueError"
    for c in query.columns:
        if c.phys_type == BOOL and c.agg_mask & (cabi.TSKV_AGG_SUM | cabi.TSKV_AGG_MEAN | cabi.TSKV_AGG_M2):
            return cabi.TSKV_ERR_INVALID_ARG
    if slide is not None:
        st = sliding_status(truth, query, slide)
        if st is not None:
            return st
        assert not has_sel and tombstones is None and "group_ids" not in extra
        return expand_aggregate(merge_truth(truth, files, query) if files is not None else truth, query, slide)
    gids, ng = extra.get("group_ids"), extra.get("n_groups")
    e, lab = extra.get("edges"), extra.get("labels")
    kw = dict(tombstones=tombstones, files=files)
    if lab is not None:
        run = (lambda: exact_aggregate_grouped_labels(truth, query, gids, ng, e, lab, **kw)) if gids is not None else \
            (lambda: exact_aggregate_labels(truth, query, e, lab, **kw))
    elif e is not None:
        run = (lambda: exact_aggregate_grouped_edges(truth, query, gids, ng, e, **kw)) if gids is not None else \
            (lambda: exact_aggregate_edges(truth, query, e, **kw))
    elif gids is not None:
        run = lambda: exact_aggregate_grouped(truth, query, gids, ng, **kw)  # noqa: E731
    else:
        run = lambda: exact_aggregate(truth, query, **kw)  # noqa: E731
    try:
        return with_m2(run, query, n_groups=ng if gids is not None else None) if has_m2 else run()
    except ReferenceError as x:
        return x.status


def case_expected(case):
    return expected(case.truth, case.query, case.extra, tombstones=case.tombstones, files=case.files)


# ---- random cases with column pairs and medians ----------------------------------------------------------------------
def operands(query):
    """(column id, type) of the pairs' operands (x0, y0, x1, ...), then the medians', then the increases'."""
    return [o for x, xt, y, yt in query.pairs for o in ((x, xt), (y, yt))] + \
        [(c.column_id, c.phys_type) for c in query.columns if c.median] + \
        [(c.column_id, c.phys_type) for c in query.columns if c.increase]


def scan_query(query):
    """The query the scan runs for one with pairs or medians (plan_operand_query): the projected columns, then every
    operand that is not one of them as a COUNT column without output."""
    cols = [PushedAggregate(c.column_id, c.phys_type, c.agg_mask) for c in query.projected()]
    for cid, pt in operands(query):
        if cid not in [c.column_id for c in cols]:
            cols.append(PushedAggregate(cid, pt, ["count"]))
    q = copy.copy(query)
    q.columns, q.pairs, q._keep = cols, [], None
    return q


def operand_columns(query):
    """-> ([(qx, qy) of every pair], [qcol of every median]): the operands' places in scan_query's columns."""
    ids = [c.column_id for c in scan_query(query).columns]
    return [(ids.index(x), ids.index(y)) for x, _, y, _ in query.pairs], \
        [ids.index(c.column_id) for c in query.columns if c.median]


# the kernels of the pairs', medians' and increases' row-by-row passes: the scan and merged-row kernels of the EXPECTED
# sets of tests/test_pair_kernel_list.py, tests/test_median_kernel_list.py and tests/test_increase_kernel_list.py, which
# hold those sets to the library (tests/test_pair_median_sweep_reference.py checks that this list is that subset)
OPERAND_KERNELS = ("k_scan_pair<false, false>", "k_scan_pair<false, true>", "k_scan_pair<true, false>",
                   "k_scan_pair<true, true>", "k_merge_pairs_rows<false>", "k_merge_pairs_rows<true>",
                   "k_scan_median<false>", "k_scan_median<true>", "k_merge_median_rows",
                   "k_scan_increase<false>", "k_scan_increase<true>", "k_merge_increase")


def merged_operands(truth, query, files, ops):
    """Whether an overlap group of two or more chunks of a selected series holds every column of `ops` (merged rows of
    those operands, which the k_merge_*_rows kernels read)."""
    if files is None:
        return False
    file_of = files_by_series(truth, files)
    for sid in (query.series_ids if query.series_ids is not None else sorted(truth)):
        cgs = truth.get(int(sid), [])
        for streams in overlap_groups(cgs, file_of.get(int(sid))):
            held = {c for st in streams for k in st for c in cgs[k][1]}
            if len(streams) >= 2 and set(ops) <= held:
                return True
    return False


def operand_kernels(wl, query, edges, truth=None, files=None):
    """The operand kernels a pass launched with work: both passes of k_scan_pair<PASS2, EDGES> when a pair's x operand
    has work-list items, k_scan_median<EDGES> when a median's operand has, k_scan_increase<EDGES> when an increase's
    operand has, k_merge_pairs_rows<PASS2> when a pair's x and y have merged rows, and k_merge_median_rows /
    k_merge_increase when a median's / an increase's operand has (merged_operands over `files`)."""
    qpairs, qmeds = operand_columns(query)
    ids = [c.column_id for c in scan_query(query).columns]
    fill = bin_fill(wl, len(ids))
    e = "true" if edges else "false"
    out = set()
    if any(fill[:, qx].sum() for qx, _ in qpairs):
        out |= {"k_scan_pair<false, %s>" % e, "k_scan_pair<true, %s>" % e}
    if any(fill[:, qc].sum() for qc in qmeds):
        out.add("k_scan_median<%s>" % e)
    if any(merged_operands(truth, query, files, (x, y)) for x, _, y, _ in query.pairs):
        out |= {"k_merge_pairs_rows<false>", "k_merge_pairs_rows<true>"}
    if any(merged_operands(truth, query, files, (c.column_id,)) for c in query.columns if c.median):
        out.add("k_merge_median_rows")
    incs = [c.column_id for c in query.columns if c.increase]
    if any(fill[:, ids.index(c)].sum() for c in incs):
        out.add("k_scan_increase<%s>" % e)
    if any(merged_operands(truth, query, files, (c,)) for c in incs):
        out.add("k_merge_increase")
    return out


def random_operand_case(index, base_seed):
    """random_case(index, base_seed) with 0-3 column pairs and 0-3 medians drawn from a stream of their own (the case's
    other draws are random_case's): pairs over the arena's numeric columns, x == y among them; medians on one column
    twice, on a projected column (the column's entry asks for it too) or on an unprojected one. At most one refusal per
    case: a case that random_case makes a refusal gets no operand; a sliding-window case gets operands only as the
    refusal "pair_sliding" / "median_sliding"; others may be "bool_pair" / "bool_median" (a BOOL operand)."""
    case = random_case(index, base_seed)
    rng = np.random.default_rng([base_seed, index, 1])
    q = case.query
    have = columns_of(case.truth)
    num = [c for c in have if COLUMNS[c] != BOOL]
    refusal = "none"
    if "slide" in case.extra:
        refusal = str(rng.choice(["pair_sliding", "median_sliding", "none"]))
    elif BOOL in [COLUMNS[c] for c in have] and rng.random() < 0.06:
        refusal = str(rng.choice(["bool_pair", "bool_median"]))
    if case.desc["refusal"] != "none" or not num or (refusal == "none" and "slide" in case.extra):
        case.desc.update(pairs=[], medians=[], operand_refusal="none")
        return case
    pick = lambda: int(rng.choice(num))  # noqa: E731
    pairs = []
    for _ in range(int(rng.integers(0, 4))):
        x = pick()
        y = x if rng.random() < 0.3 else pick()
        pairs.append((x, COLUMNS[x], y, COLUMNS[y]))
    meds = []
    for _ in range(int(rng.integers(0, 4))):
        c = meds[-1] if meds and rng.random() < 0.25 else pick()
        meds.append(c)
    if refusal in ("pair_sliding", "bool_pair") and not pairs:
        x = pick()
        pairs.append((x, COLUMNS[x], x, COLUMNS[x]))
    if refusal in ("median_sliding", "bool_median") and not meds:
        meds.append(pick())
    if refusal == "bool_pair":
        k = int(rng.integers(0, len(pairs)))
        x, xt, y, yt = pairs[k]
        pairs[k] = (4, BOOL, y, yt) if rng.random() < 0.5 else (x, xt, 4, BOOL)
    if refusal == "bool_median":
        meds[int(rng.integers(0, len(meds)))] = 4
    q.pairs = pairs
    for c in meds:
        entry = [e for e in q.columns if e.column_id == c and e.agg_mask and not e.median]
        if entry and rng.random() < 0.5:
            entry[0].median = True  # the projected entry asks for the median as well
        else:
            q.columns.append(PushedAggregate(c, COLUMNS[c], ["median"]))
    case.desc.update(pairs=[(x, y) for x, _, y, _ in pairs], medians=[c.column_id for c in q.columns if c.median],
                     operand_refusal=refusal)
    return case


# ---- random cases with counter increases -------------------------------------------------------------------------------
def selected_slots(truth, query):
    """The series a scan selects: series_ids, or else every series of the page set."""
    return list(query.series_ids) if query.series_ids is not None else sorted(truth)


def increase_status(truth, query, extra):
    """The status the scan refuses a query with increases with (None: accepted), in the order the engine and
    validate_query check (cnosdb_b200/csrc/tskv_gpu.cu, the increase checks at the end of validate_query):
      1. a sliding window: the engine's ValueError, before the library is called;
      2. an operand of type BOOL (a pair's, a median's or an increase's): TSKV_ERR_INVALID_ARG (the operand checks
         come before every grouping check);
      3. bucket labels: TSKV_ERR_UNSUPPORTED (date_part cells are not monotone in time);
      4. a tag group map under which two selected slots share a group: TSKV_ERR_UNSUPPORTED;
      5. no group map and no GROUP BY series over more than one selected slot ("selected": series_ids, or else every
         series of the page set): TSKV_ERR_UNSUPPORTED.
    A cell of an accepted query holds rows of one series."""
    if extra.get("slide") is not None:
        return "ValueError"
    if BOOL in [pt for _, pt in operands(query)]:
        return cabi.TSKV_ERR_INVALID_ARG
    if extra.get("labels") is not None:
        return cabi.TSKV_ERR_UNSUPPORTED
    gids = extra.get("group_ids")
    n_slots = len(selected_slots(truth, query))
    if gids is not None:
        if len(set(int(g) for g in gids[:n_slots])) < n_slots:
            return cabi.TSKV_ERR_UNSUPPORTED
    elif not query.group_by_series and n_slots > 1:
        return cabi.TSKV_ERR_UNSUPPORTED
    return None


INC_SHAPES = ("series", "tags", "edges", "one")


def random_increase_case(index, base_seed):
    """random_case(index, base_seed) with 1-4 increases drawn from a stream of their own (random_case's draws are
    unchanged): increases of numeric columns, duplicates and unprojected columns among them, sometimes with a pair or a
    median. With probability 0.7 the case is regrouped into a shape whose cells hold one series (INC_SHAPES: GROUP BY
    series; a tag map of one selected series per group; edges with GROUP BY series; one selected series, bucketed or
    not); otherwise it keeps random_case's grouping and increase_status says whether the scan refuses it. A case that
    random_case makes a refusal gets no increase; a few cases turn one increase into a BOOL operand (refused)."""
    case = random_case(index, base_seed)
    rng = np.random.default_rng([base_seed, index, 2])
    q = case.query
    have = columns_of(case.truth)
    num = [c for c in have if COLUMNS[c] != BOOL]
    if case.desc["refusal"] != "none" or not num:
        case.desc.update(increases=[], shape="kept", increase_refusal="none")
        return case
    incs = [int(rng.choice(num)) for _ in range(int(rng.integers(1, 5)))]
    if len(incs) > 1 and rng.random() < 0.3:
        incs[-1] = incs[0]  # (a duplicate)
    bool_op = BOOL in [COLUMNS[c] for c in have] and rng.random() < 0.05
    if bool_op:
        incs[int(rng.integers(0, len(incs)))] = 4
    if rng.random() < 0.25:
        x, y = int(rng.choice(num)), int(rng.choice(num))
        q.pairs = [(x, COLUMNS[x], y, COLUMNS[y])]
    if rng.random() < 0.25:
        c = int(rng.choice(num))
        q.columns.append(PushedAggregate(c, COLUMNS[c], ["median"]))
    for c in incs:
        entry = [e for e in q.columns if e.column_id == c and e.agg_mask and not e.increase]
        if entry and rng.random() < 0.5:
            entry[0].increase = True  # the projected entry asks for the increase as well
        else:
            q.columns.append(PushedAggregate(c, COLUMNS[c], ["increase"]))
    shape = str(rng.choice(INC_SHAPES)) if rng.random() < 0.7 else "kept"
    if shape != "kept":
        lo, hi = span(case.truth)
        step = case.desc["step"]
        for k in ("slide", "edges", "labels", "group_ids", "n_groups"):
            case.extra.pop(k, None)
        w = int(rng.choice([37, 100, 1000])) * step
        origin = int(rng.integers(-w, w))
        fbs, nb = bucket_spec(lo, hi, w, origin)
        q.width, q.origin, q.first_bucket_start, q.n_buckets, q.group_by_series = w, origin, fbs, nb, False
        sids = sorted(case.truth)
        if shape == "series":
            q.group_by_series = True
        elif shape == "tags":
            n_slots = len(selected_slots(case.truth, q))
            n_groups = n_slots + int(rng.integers(0, 3))
            case.extra["n_groups"] = n_groups
            case.extra["group_ids"] = rng.permutation(n_groups)[:n_slots].astype(np.uint32)
        elif shape == "edges":
            e = random_edges(rng, lo, hi, int(rng.integers(1, 60)))
            case.extra["edges"] = e
            q.width, q.origin, q.first_bucket_start, q.n_buckets, q.group_by_series = 0, 0, 0, e.size - 1, True
        else:
            q.series_ids = np.array([sids[int(rng.integers(0, len(sids)))]], dtype=np.uint32)
            if rng.random() < 0.5:
                q.width, q.origin, q.first_bucket_start, q.n_buckets = 0, 0, 0, 1
        q._keep = None
    case.desc.update(increases=incs, shape=shape, increase_refusal="bool_increase" if bool_op else "none",
                     pairs=[(x, y) for x, _, y, _ in q.pairs], medians=[c.column_id for c in q.columns if c.median],
                     inc_width=q.width, inc_n_buckets=q.n_buckets, inc_group_by_series=q.group_by_series,
                     inc_series_ids=None if q.series_ids is None else q.series_ids.tolist(),
                     inc_n_groups=case.extra.get("n_groups"))
    return case
