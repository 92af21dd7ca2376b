"""Simple8b integer pages whose values all lie in [-2^31, 2^31) (i64) or [0, 2^31) (u64) ("narrow" pages, flagged at upload
from the decoded values) are accumulated in 32-bit arithmetic by the fused scan. Every output must equal the wide arithmetic's:
COUNT / SUM / MIN / MAX bit for bit against the oracle, and COUNT / SUM / MIN / MAX / MEAN bit for bit against the exact
reference (MEAN = float(S) / float(n)). The pages sit right at the narrow range's edges (INT32_MIN / INT32_MAX and one
past them, u64 2^31 - 1 / 2^31 / above 2^63), alternate between INT32_MIN and INT32_MAX (60-bit simple8b codes), hold
nulls, mix with wide pages in one warp's chunk, and sum past 2^32 in one cell. They go through the uniform bucket
schedule, the segment loop and the simple8b-timestamp loop, with one and three parts per page, time ranges, field
predicates, tombstones, GROUP BY tags, sliding windows and a host-resident page set; a truncated page must fail like the
oracle says."""
import numpy as np
import pytest

from cnosdb_b200 import cabi, datagen
from cnosdb_b200.engine import TskvError
from oracle import pyoracle as orc
from tests.group_reference import exact_aggregate_grouped
from tests.helpers import assert_matches_exact, exact_aggregate, make_query
from tests.sliding_reference import pane_aggregate
from tests.test_gpu_parity import random_tombstones

pytestmark = pytest.mark.gpu

I32_MIN, I32_MAX = -2**31, 2**31 - 1
FIELDS = ((1, cabi.TSKV_PT_I64), (3, cabi.TSKV_PT_U64))
AGGS = ("count", "sum", "min", "max", "mean")
T0, STEP = 1_000_000_000_000, 1000
N_SERIES, ROWS, SHORT_ROWS = 256, 700, 100
W = 16 * STEP


def i64_values(rng, sid, m):
    walk = np.cumsum(rng.integers(-3, 4, m)).astype(np.int64)
    k = sid % 8
    if k == 0:  # TSBS-like percentages
        return np.clip(50 + walk, 0, 100)
    if k == 1:  # exactly at the edges: narrow
        v = np.clip(walk * 2**27, I32_MIN, I32_MAX)
        v[m // 3], v[m // 2] = I32_MIN, I32_MAX
        return v
    if k == 2:  # alternating INT32_MIN / INT32_MAX: 34-bit zig-zag codes in 60-bit simple8b words
        return np.where(np.arange(m) % 2 == 0, I32_MIN, I32_MAX).astype(np.int64)
    if k == 3:  # one past INT32_MAX: wide
        v = np.clip(I32_MAX - 40 + walk, I32_MIN, I32_MAX)
        v[m // 2] = I32_MAX + 1
        return v
    if k == 4:  # one past INT32_MIN: wide
        v = np.clip(I32_MIN + 40 + walk, I32_MIN, I32_MAX)
        v[m // 4] = I32_MIN - 1
        return v
    if k == 5:  # near INT32_MAX: a cell's sum passes 2^32 (narrow)
        return np.clip(I32_MAX - 1000 + walk, I32_MIN, I32_MAX)
    if k == 6:  # near INT32_MIN (narrow)
        return np.clip(I32_MIN + 1000 + walk, I32_MIN, I32_MAX)
    return walk * 2**34  # wide everywhere


def u64_values(rng, sid, m):
    walk = np.cumsum(rng.integers(0, 4, m)).astype(np.uint64)
    k = sid % 5
    if k == 0:
        return walk % np.uint64(101)
    if k == 1:  # up to 2^31 - 1: narrow
        v = np.uint64(2**31 - 1) - walk % np.uint64(5000)
        v[m // 2] = 2**31 - 1
        return v
    if k == 2:  # one value at 2^31: wide
        v = np.uint64(2**31 - 1) - walk % np.uint64(5000)
        v[m // 3] = 2**31
        return v
    if k == 3:  # above 2^63
        return np.uint64(2**63 + 17) + walk
    return np.uint64(2**64 - 1) - walk  # wide, though each value sign-extends from its low 32 bits as an i64


def timestamps(rng, sid, m):
    """The first half share their rows (uniform schedule), the next quarter start sid % 7 rows later (segment loop), the
    last quarter are jittered (simple8b time pages)."""
    if sid < N_SERIES // 2:
        return T0 + np.arange(m, dtype=np.int64) * STEP
    if sid < 3 * N_SERIES // 4:
        return T0 + (sid % 7 + np.arange(m, dtype=np.int64)) * STEP
    return T0 + np.arange(m, dtype=np.int64) * STEP + rng.integers(0, STEP // 2, m)


NARROW_I64, NARROW_U64 = (0, 1, 2, 5, 6), (0, 1)


def build(seed, narrow_only=False, cuts=1):
    """narrow_only: every page narrow (the bins run the kernels that hold the 32-bit arithmetic only); otherwise narrow
    and wide pages share the bins (kernels that choose per chunk). cuts: column groups per series (its rows cut into
    consecutive runs)."""
    rng = np.random.default_rng(seed)
    b = datagen.ArenaBuilder()
    truth = {}
    for sid in range(N_SERIES):
        m = SHORT_ROWS if sid % 9 == 4 else ROWS  # pages of <= 128 rows have no restart points
        ts = timestamps(rng, sid, m)
        ik, uk = (NARROW_I64[sid % 5], NARROW_U64[sid % 2]) if narrow_only else (sid, sid)
        iv, uv = i64_values(rng, ik, m), u64_values(rng, uk, m)
        valid = rng.random(m) >= 0.3 if sid % 13 == 6 else np.ones(m, dtype=bool)
        truth[sid] = []
        for r in np.array_split(np.arange(m), cuts):
            vv = None if valid[r].all() else valid[r]
            b.add_column_group(sid, ts[r], [(1, cabi.TSKV_PT_I64, iv[r], vv), (3, cabi.TSKV_PT_U64, uv[r], vv)])
            truth[sid].append((ts[r], {1: (iv[r], valid[r]), 3: (uv[r], valid[r])}))
    arena, descs = b.finish()
    return arena, descs, truth


@pytest.fixture(scope="module")
def narrow_set():
    return build(11)


@pytest.fixture(scope="module")
def narrow_cut_set():
    return build(11, cuts=3)


@pytest.fixture(scope="module")
def all_narrow_set():
    return build(12, narrow_only=True)


def grid(n_rows=ROWS + 8):
    return dict(width=W, first_bucket_start=T0 - (T0 % W), n_buckets=(T0 % W + n_rows * STEP) // W + 1)


def queries():
    pred = [(1, cabi.TSKV_PT_I64, ">=", 0)]
    return [
        ("bucket", make_query(FIELDS, AGGS, **grid())),
        ("range", make_query(FIELDS, AGGS, time_ranges=[(T0 + 37 * STEP + 1, T0 + 555 * STEP)], **grid())),
        ("predicate", make_query(FIELDS, AGGS, predicates=pred, **grid())),
        ("unbucketed", make_query(FIELDS, AGGS)),
        ("subset", make_query(FIELDS, AGGS, series_ids=np.arange(1, N_SERIES, 3, dtype=np.uint32), **grid())),
    ]


def assert_int_equal(got, exp, what):
    """Every output of two integer-only results, bit for bit."""
    assert got.names == exp.names
    for j, (col, agg) in enumerate(got.names):
        assert (got.validity[j] == exp.validity[j]).all(), (what, col, agg)
        bad = np.nonzero(got.values[j] != exp.values[j])[0]
        assert bad.size == 0, "%s col %s %s differs at %s" % (what, col, agg, bad[:5])


def assert_oracle_equal(got, ora, what):
    """COUNT / SUM / MIN / MAX bit for bit against the oracle (its MEAN divides an f64 running sum)."""
    for j, (col, agg) in enumerate(got.names):
        if agg == "mean":
            continue
        assert (got.validity[j] == ora.validity[j]).all(), (what, col, agg)
        bad = np.nonzero(got.values[j] != ora.values[j])[0]
        assert bad.size == 0, "%s col %s %s differs from the oracle at %s" % (what, col, agg, bad[:5])


def mixed_chunks(arena, descs, truth):
    """Where a scan of every page puts narrow and wide pages into one 32-page chunk, restated from the arrays. Every
    simple8b value page here has at most 1024 rows, so its bin is the short-page bin of its time page's codec (run-length
    or simple8b). The work list holds a bin's pages column by column (the query's column order), each column's wide
    pages before its narrow ones, and cuts the bin into chunks of 32 from its start: a chunk mixes the two kinds where
    a wide / narrow boundary falls off a multiple of 32. Returns [(time codec, boundary)]."""
    def int_kind(d):  # integer encoding of the page's data (page.rs framing): 1 = simple8b, 2 = run-length
        off = int(d["offset"])
        return int(arena[off + 16 + int.from_bytes(arena[off:off + 4].tobytes(), "big") + 1]) >> 4

    groups = [(ts, cols) for cgs in truth.values() for ts, cols in cgs]
    tps = np.nonzero(descs["phys_type"] == cabi.TSKV_PT_TIME)[0]
    assert len(tps) == len(groups)
    count = {}  # (time codec, column, narrow) -> pages
    for k, (ts, cols) in enumerate(groups):
        tk = int_kind(descs[tps[k]])
        for p in range(tps[k] + 1, tps[k + 1] if k + 1 < len(tps) else len(descs)):
            d = descs[p]
            if int_kind(d) != 1:
                continue  # a run-length value page: a bin of its own, never narrow
            assert int(d["num_values"]) <= 1024
            v, valid = cols[int(d["column_id"])]
            v = v[valid]
            narrow = bool((v <= I32_MAX).all() and (v >= (I32_MIN if v.dtype == np.int64 else 0)).all())
            key = (tk, int(d["column_id"]), narrow)
            count[key] = count.get(key, 0) + 1
    out = []
    for tk in (1, 2):
        pos, last = 0, None
        for col, _ in FIELDS:
            for narrow in (False, True):
                n = count.get((tk, col, narrow), 0)
                if n and last is not None and last != narrow and pos % 32:
                    out.append((tk, pos))
                if n:
                    pos, last = pos + n, narrow
    return out


@pytest.mark.parametrize("env", ["parts1", "parts3", "cut"])
def test_narrow_pages_are_exact(engine, narrow_set, narrow_cut_set, env, monkeypatch):
    """parts1 / parts3: pages whole or cut in three at restart points; cut: every series cut into three column groups,
    which puts wide / narrow boundaries inside 32-page chunks (mixed_chunks), so those chunks take the per-chunk choice."""
    arena, descs, truth = narrow_cut_set if env == "cut" else narrow_set
    monkeypatch.setenv("TSKV_PARTS", "3" if env == "parts3" else "1")
    if env == "cut":
        assert mixed_chunks(arena, descs, truth)
    pages = engine.upload_pages(arena, descs)
    for name, q in queries():
        got = engine.scan_aggregate(pages, q)
        assert_matches_exact(got, exact_aggregate(truth, q), what="%s %s" % (env, name))
        assert_oracle_equal(got, orc.scan_aggregate(arena, descs, q), "%s %s" % (env, name))
    pages.close()


@pytest.mark.parametrize("parts", ["1", "3"])
def test_all_narrow_page_set(engine, all_narrow_set, parts, monkeypatch):
    arena, descs, truth = all_narrow_set
    monkeypatch.setenv("TSKV_PARTS", parts)
    pages = engine.upload_pages(arena, descs)
    host = engine.upload_pages(arena, descs, host_resident=True)
    for name, q in queries():
        got = engine.scan_aggregate(pages, q)
        assert_matches_exact(got, exact_aggregate(truth, q), what="all narrow %s %s" % (parts, name))
        assert_oracle_equal(got, orc.scan_aggregate(arena, descs, q), "all narrow %s %s" % (parts, name))
        assert_int_equal(got, engine.scan_aggregate(host, q), "all narrow vs host-resident " + name)
    host.close()
    pages.close()


def test_mean_sum_passes_2_32(engine, narrow_set):
    """Series near INT32_MAX (narrow) summed into few cells: S passes 2^32 in the buckets, and 10^13 unbucketed."""
    arena, descs, truth = narrow_set
    ids = np.arange(5, N_SERIES, 8, dtype=np.uint32)
    pages = engine.upload_pages(arena, descs)
    for q in (make_query(FIELDS[:1], AGGS, series_ids=ids, **grid()), make_query(FIELDS[:1], AGGS, series_ids=ids)):
        exp = exact_aggregate(truth, q)
        assert max(S for S, _ in exp.exact_sums[1].values()) > 2**32
        assert_matches_exact(engine.scan_aggregate(pages, q), exp, what="mean > 2^32")
    pages.close()


def test_tombstones(engine, narrow_set):
    arena, descs, _ = narrow_set
    rng = np.random.default_rng(5)
    tombs = random_tombstones(rng, descs, T0, T0 + ROWS * STEP)
    pages = engine.upload_pages(arena, descs)
    pages.set_tombstones(tombs)
    for name, q in queries()[:3]:
        got = engine.scan_aggregate(pages, q)
        ora = orc.scan_aggregate(arena, descs, q, tombstones=tombs)
        assert_oracle_equal(got, ora, "tombstones " + name)
    pages.close()


def test_group_by_tags_and_sliding_windows(engine, narrow_set):
    arena, descs, truth = narrow_set
    pages = engine.upload_pages(arena, descs)
    q = make_query(FIELDS, AGGS, **grid())
    gids = (np.arange(N_SERIES) * 7 % 5).astype(np.uint32)
    got = engine.scan_aggregate(pages, q, group_ids=gids, n_groups=5)
    assert_matches_exact(got, exact_aggregate_grouped(truth, q, gids, 5), what="group by tags")
    window, slide = 4 * W, W
    g = grid()
    sq = make_query(FIELDS, AGGS, width=window, first_bucket_start=g["first_bucket_start"] - 3 * W, n_buckets=g["n_buckets"] + 3)
    got = engine.scan_aggregate(pages, sq, slide=slide)
    assert_matches_exact(got, pane_aggregate(truth, sq, slide), what="sliding windows")
    pages.close()


def test_host_resident_page_set(engine, narrow_set):
    """Host-resident page sets carry no narrow flags: the wide arithmetic gives the same outputs."""
    arena, descs, truth = narrow_set
    dev = engine.upload_pages(arena, descs)
    host = engine.upload_pages(arena, descs, host_resident=True)
    for name, q in queries():
        a, b = engine.scan_aggregate(dev, q), engine.scan_aggregate(host, q)
        assert_int_equal(a, b, "host-resident " + name)
        assert_matches_exact(b, exact_aggregate(truth, q), what="host-resident " + name)
    host.close()
    dev.close()


@pytest.mark.parametrize("rows", [SHORT_ROWS, ROWS])
def test_truncated_page_fails_like_the_oracle(engine, rows, monkeypatch):
    """A simple8b page of narrow values that lacks its last word: the same status and page as the oracle (and as the
    wide arithmetic, whose cursor consumes the same words), next to intact narrow pages."""
    rng = np.random.default_rng(rows)
    b = datagen.ArenaBuilder()
    for sid in range(40):
        ts = T0 + np.arange(rows, dtype=np.int64) * STEP
        v = np.clip(50 + np.cumsum(rng.integers(-3, 4, rows)), 0, 100).astype(np.int64)
        if sid != 17:
            b.add_column_group(sid, ts, [(1, cabi.TSKV_PT_I64, v, None)])
            continue
        data = datagen.encode_integers(v)
        assert data[1] >> 4 == 1  # simple8b
        b.add_page(datagen.build_page(datagen.encode_timestamps(ts), rows), sid, 0, cabi.TSKV_PT_TIME, rows)
        b.add_page(datagen.build_page(data[:-8], rows), sid, 1, cabi.TSKV_PT_I64, rows)
    arena, descs = b.finish()
    q = make_query(FIELDS[:1], AGGS, **grid())
    with pytest.raises(orc.OracleError) as oe:
        orc.scan_aggregate(arena, descs, q)
    pages = engine.upload_pages(arena, descs)
    for parts in ("1", "3"):
        monkeypatch.setenv("TSKV_PARTS", parts)
        with pytest.raises(TskvError) as ge:
            engine.scan_aggregate(pages, q)
        assert ge.value.status == oe.value.status and ge.value.page == 2 * 17 + 1, (parts, ge.value.status, ge.value.page)
    pages.close()
