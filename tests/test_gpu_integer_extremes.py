"""Integer SUM / MEAN through every carry of the fused scan's accumulators, checked against exact Python-int sums:
values near the i64 / u64 limits (simple8b walks, cancelling blocks of +-2^62..2^63, constant run-length pages, raw
pages), 2 000 series into a few cells (the table atomics carry into the high word), and 102 400-row pages of INT64_MAX.
SUM must equal S mod 2^64 and MEAN float(S) / float(n), bit for bit; COUNT / MIN / MAX exactly. f64 columns (magnitudes
up to 1e290, cancelling +-1e16 blocks, +-0.0) stay within the order-free bound of their exact sum. The data runs through
the uniform bucket schedule, the segment loop, the FIRST / LAST kernels, group_by_series, the
global-atomics table, the overlap merge and a two-shard exchange."""
from fractions import Fraction

import numpy as np
import pytest

from cnosdb_b200 import cabi, datagen
from oracle import pyoracle as orc
from tests.helpers import ALL_AGGS, I64_MAX, I64_MIN, assert_matches_exact, exact_aggregate, make_query

pytestmark = pytest.mark.gpu

FIELDS = ((1, cabi.TSKV_PT_I64), (2, cabi.TSKV_PT_F64), (3, cabi.TSKV_PT_U64))
AGGS = ("count", "sum", "min", "max", "mean")
T0, STEP = 1_000_000_007, 1000
N_SERIES, ROWS = 2000, 64
W = 16 * STEP  # 4 to 5 buckets per page
BIG_IDS = range(N_SERIES, N_SERIES + 4)  # 102 400-row pages of INT64_MAX
BIG_ROWS = 102_400
BY_SERIES_IDS = np.r_[0:40, 1000:1016, N_SERIES:N_SERIES + 4].astype(np.uint32)  # (keeps the cell count small)


def i64_values(rng, sid, m):
    walk = np.cumsum(rng.integers(0, 50, m)).astype(np.int64)
    k = sid % 6
    if k == 0:
        return np.int64(I64_MAX) - walk, None
    if k == 1:
        return np.int64(I64_MIN) + walk, None
    if k == 2:  # cancelling blocks: S is small, the partial sums are huge
        x = rng.integers(2**62, 2**63 - 1, m // 2 + 1, dtype=np.int64)
        return np.concatenate([x, -x])[:m], None
    if k == 3:
        return np.full(m, I64_MAX, dtype=np.int64), None  # constant: a run-length value page
    if k == 4:
        return np.full(m, I64_MIN, dtype=np.int64), None
    return np.int64(I64_MAX) - walk, datagen.encode_raw  # raw


def u64_values(rng, sid, m):
    walk = np.cumsum(rng.integers(0, 50, m)).astype(np.uint64)
    k = sid % 3
    if k == 0:
        return np.uint64(2**64 - 1) - walk
    if k == 1:
        return np.uint64(2**63 - 700) + walk  # straddles 2^63
    return np.full(m, 2**64 - 1, dtype=np.uint64)


def f64_values(rng, sid, m):
    k = sid % 3
    if k == 0:
        return rng.choice([-1, 1], m) * 10.0 ** rng.uniform(-300, 290, m)
    if k == 1:
        x = 1e16 * (1 + rng.random(m // 2 + 1))
        return np.concatenate([x, -x])[:m] + rng.integers(-3, 4, m)
    return rng.choice([-0.0, 0.0], m)


def build(seed, ids, rows_of, start_of, nulls=True):
    rng = np.random.default_rng(seed)
    b = datagen.ArenaBuilder()
    truth = {}
    for sid in ids:
        m = rows_of(sid)
        ts = T0 + (start_of(sid) + np.arange(m, dtype=np.int64)) * STEP
        iv, ienc = i64_values(rng, sid, m)
        if sid in BIG_IDS:
            iv, ienc = np.full(m, I64_MAX, dtype=np.int64), None
        uv, fv = u64_values(rng, sid, m), f64_values(rng, sid, m)
        valid = rng.random(m) >= 0.25 if (nulls and sid % 11 == 5) else np.ones(m, dtype=bool)
        vv = None if valid.all() else valid
        b.add_column_group(sid, ts, [(1, cabi.TSKV_PT_I64, iv, vv, ienc), (2, cabi.TSKV_PT_F64, fv, vv),
                                     (3, cabi.TSKV_PT_U64, uv, vv)])
        truth[sid] = [(ts, {1: (iv, valid), 2: (fv, valid), 3: (uv, valid)})]
    arena, descs = b.finish()
    return arena, descs, truth


@pytest.fixture(scope="module")
def extremes():
    # the first half share their timestamps (uniform schedule), the second half start sid % 7 rows later (segment loop)
    ids = list(range(N_SERIES)) + list(BIG_IDS)
    return build(7, ids, lambda s: BIG_ROWS if s in BIG_IDS else ROWS,
                 lambda s: 0 if (s < N_SERIES // 2 or s in BIG_IDS) else s % 7)


def queries(nb_rows):
    grid = dict(width=W, first_bucket_start=T0 - (T0 % W), n_buckets=(T0 % W + nb_rows * STEP) // W + 1)
    return [
        ("bucket", make_query(FIELDS, AGGS, **grid)),
        ("bucket+sel", make_query(FIELDS, ALL_AGGS, **grid)),
        ("by_series", make_query(FIELDS, AGGS, group_by_series=True, series_ids=BY_SERIES_IDS, **grid)),
        ("unbucketed", make_query(FIELDS, AGGS)),
        ("range", make_query(FIELDS, AGGS, time_ranges=[(T0 + 3 * STEP, T0 + 50_000 * STEP)], **grid)),
    ]


@pytest.mark.parametrize("env", ["default", "global_atomics", "parts3"])
def test_integer_extremes_are_exact(engine, extremes, env, monkeypatch):
    arena, descs, truth = extremes
    monkeypatch.setenv("TSKV_PARTS", "3" if env == "parts3" else "1")
    if env == "global_atomics":
        monkeypatch.setenv("TSKV_SMEM_TABLE_KB", "0")
    pages = engine.upload_pages(arena, descs)
    for name, q in queries(BIG_ROWS):
        exp = exact_aggregate(truth, q)
        got = engine.scan_aggregate(pages, q)
        assert_matches_exact(got, exp, what="%s %s" % (env, name))
        if name == "bucket+sel":
            ora = orc.scan_aggregate(arena, descs, q)
            for j, (col, agg) in enumerate(got.names):
                if agg in ("first", "last"):
                    assert (got.validity[j] == ora.validity[j]).all() and (got.values[j] == ora.values[j]).all(), (env, col, agg)
    pages.close()


def test_overlap_merge_keeps_exact_sums(engine):
    """Two chunk files of one series whose time ranges overlap (rows interleave, none collide): the merge kernel's
    accumulation of the merged rows."""
    rng = np.random.default_rng(3)
    b = datagen.ArenaBuilder()
    cgs, files = [], []
    for f in range(2):
        for part in range(2):
            m = 300
            ts = T0 + (2 * (np.arange(m, dtype=np.int64) + part * m) + f) * STEP  # file 0 even rows, file 1 odd rows
            iv, _ = i64_values(rng, 2 + f, m)  # cancelling blocks / constant INT64_MAX
            uv, fv = u64_values(rng, f, m), f64_values(rng, f, m)
            ok = np.ones(m, dtype=bool)
            b.add_column_group(9, ts, [(1, cabi.TSKV_PT_I64, iv, None), (2, cabi.TSKV_PT_F64, fv, None),
                                       (3, cabi.TSKV_PT_U64, uv, None)])
            cgs.append((ts, {1: (iv, ok), 2: (fv, ok), 3: (uv, ok)}))
            files.append(f + 1)
    arena, descs = b.finish()
    truth = {9: cgs}
    pages = engine.upload_pages(arena, descs)
    pages.set_chunk_files(files)
    for name, q in queries(4 * 300):
        exp = exact_aggregate(truth, q)
        assert_matches_exact(engine.scan_aggregate(pages, q), exp, what="overlap merge " + name)
        if name == "bucket+sel":
            ora = orc.scan_aggregate(arena, descs, q, chunk_files=files)
            got = engine.scan_aggregate(pages, q)
            for j, (col, agg) in enumerate(got.names):
                if agg in ("first", "last"):
                    assert (got.values[j] == ora.values[j]).all(), (col, agg)
    pages.close()


def test_two_shard_exchange_of_extreme_sums(engine, extremes):
    """Two contiguous series shards scanned separately and merged like an all-gather on one device. Each rank exports
    its integer MEAN sum as f64 before the merge, so MEAN is only held to |got * n - S| <= 2^-52 * sum|S_r| + 2^-53 * |S|
    (S_r: the ranks' exact sums); COUNT / SUM / MIN / MAX stay exact."""
    import torch
    from cnosdb_b200.parallel import device_tensor
    _, _, truth = extremes
    ids = sorted(truth)
    half = len(ids) // 2
    q = queries(BIG_ROWS)[0][1]
    q.series_ids = np.array(ids, dtype=np.uint32)
    exp = exact_aggregate(truth, q)
    dev = torch.device("cuda", engine.device)
    scans, regions, keep, shard_sums = [], [], [], []
    for r, part in enumerate((ids[:half], ids[half:])):
        sub = {s: truth[s] for s in part}
        b = datagen.ArenaBuilder()  # the shard's pages, from the same rows
        for s in part:
            ts, cols = truth[s][0]
            b.add_column_group(s, ts, [(c, pt, cols[c][0], None if cols[c][1].all() else cols[c][1]) for c, pt in FIELDS])
        arena, descs = b.finish()
        pages = engine.upload_pages(arena, descs)
        s = engine.prepare(pages, q)
        s.run()
        ptr, words = s.exchange_view()
        regions.append(device_tensor(ptr, words, torch.int64, dev).clone())
        scans.append(s)
        keep.append(pages)
        shard_sums.append(exact_aggregate(sub, q).exact_sums)
    gathered = torch.cat(regions)
    torch.cuda.synchronize()
    for s in scans:
        s.merge_gathered(gathered.data_ptr(), 2)
        got = s.finalize()
        assert_matches_exact(got, exp, what="2-shard exchange", int_mean=False)
        for j, (col, agg) in enumerate(got.names):
            if agg != "mean" or col == 2:
                continue
            for cell, (S, n) in exp.exact_sums[col].items():
                sr = sum(abs(sh[col].get(cell, (0, 0))[0]) for sh in shard_sums)
                g = Fraction(float(got.values[j].view(np.float64)[cell]))
                assert abs(g * n - S) <= Fraction(sr, 2**52) + Fraction(abs(S), 2**53), (col, cell)
        s.close()
    for pages in keep:
        pages.close()
