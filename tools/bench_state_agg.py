"""The cost of compact_state_agg(time, x) and of state_agg(time, x) in alternating runs on one GPU: MEAN only
(`mean`), MEAN plus the i64 column's (column 1) compact state agg (`state_i64`: its duration map) and MEAN plus its state
agg (`periods_i64`: the map and the periods, TSKV_STATE_PERIODS), ms per step (one enqueue of the prepared scan followed
by its sync):

  c4/one_series     C4 (bench.py), its first selected series with an i64 column alone, unbucketed (a state agg cell
                    holds one series)
  c4/series         C4 GROUP BY series on its tumbling grid, over its selected series that hold the i64 column (the
                    other half of C4's series has no i64 page, which the scan refuses: their rows would be NULL states)
  runs/series       a page set of its own: i64 states 0..4 in runs of about 100 rows (geometric lengths), built with
                    ArenaBuilder here; GROUP BY series on 1-minute buckets

C4's i64 column is a random walk, so nearly every row starts a run of its own: the worst case, about one duration record
per row. The run-structured set makes about one per 100 rows.

  python tools/bench_state_agg.py [--series N] [--run-series S] [--run-rows R] [--steps K] [--warmup W] [--rounds R] [--out DIR]

Prints one JSON line: ms per step of each variant (median, min, max over the rounds), the card's name and power limit,
the counters, the map entries, periods and selected rows of each state agg variant, and whether the MEAN outputs of the
state agg variants equal the `mean` variant's (bit for bit; f64 within 1e-12 relative) and the periods variant's map
entries the compact variant's. Exits non-zero otherwise. Writes the JSON to DIR/bench_state_agg.json."""
import argparse
import json
import os
import statistics
import sys

import numpy as np

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(ROOT))
sys.path.insert(0, ROOT)

import bench  # noqa: E402
from bench_bucket_edges import time_steps  # noqa: E402
from cnosdb_b200 import cabi, datagen  # noqa: E402
from cnosdb_b200.engine import Engine, PushedAggregate, QueryOption  # noqa: E402

MIN = 60_000_000_000


VARIANTS = {"mean": [], "state_i64": ["compact_state_agg"], "periods_i64": ["state_agg"]}


def c4_variant(q, variant, grid, with_i64):
    cols = [PushedAggregate(c.column_id, c.phys_type, ["mean"] + (VARIANTS[variant] if c.column_id == 1 else []))
            for c in q.columns]
    kw = dict(series_ids=q.series_ids, time_ranges=q.time_ranges, origin=q.origin, width=q.width,
              first_bucket_start=q.first_bucket_start, n_buckets=q.n_buckets,
              predicates=[(c, pt, op, v) for c, pt, op, v in q.predicates])
    if grid == "one_series":
        kw.update(series_ids=with_i64[:1], width=0, origin=0, first_bucket_start=0, n_buckets=1)
    else:
        kw.update(series_ids=with_i64, group_by_series=True)
    return QueryOption(cols, **kw)


def run_arena(n_series, n_rows, seed=7):
    """i64 states 0..4 in geometric runs of mean 100 rows, one f64 column beside them, 1 s apart."""
    rng = np.random.default_rng(seed)
    b = datagen.ArenaBuilder()
    t0 = 1_700_000_000_000_000_000
    ts = t0 + np.arange(n_rows, dtype=np.int64) * 1_000_000_000
    runs = 0
    for sid in range(n_series):
        lens = rng.geometric(0.01, n_rows // 50 + 10)
        lens = lens[: np.searchsorted(np.cumsum(lens), n_rows) + 1]
        v = np.repeat(rng.integers(0, 5, lens.size).astype(np.int64), lens)[:n_rows]
        runs += int(np.count_nonzero(np.diff(v)) + 1)
        f = rng.random(n_rows)
        for k in range(0, n_rows, 4096):  # column groups of 4096 rows
            b.add_column_group(sid, ts[k:k + 4096], [(1, cabi.TSKV_PT_I64, v[k:k + 4096], None), (2, cabi.TSKV_PT_F64, f[k:k + 4096], None)])
    a, d = b.finish()
    return a, d, t0, int(ts[-1]), runs


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--series", type=int, default=bench.WORKLOADS["C4"].default_series)
    ap.add_argument("--run-series", type=int, default=1000)
    ap.add_argument("--run-rows", type=int, default=8192)
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()

    engine = Engine(0)
    g = bench.generate_shard(args.series, 0, 1)
    c4 = engine.upload_pages(g.arena, g.descs)
    base = bench.make_query(bench.WORKLOADS["C4"].select(args.series))
    d = g.descs
    has_i64 = np.unique(d["series_id"][(d["column_id"] == 1) & (d["phys_type"] == cabi.TSKV_PT_I64)])
    with_i64 = np.intersect1d(base.series_ids, has_i64).astype(np.uint32)
    ra, rd, r_lo, r_hi, n_runs = run_arena(args.run_series, args.run_rows)
    rp = engine.upload_pages(ra, rd)
    queries = {}
    for grid in ("one_series", "series"):
        for name in VARIANTS:
            queries["c4/%s/%s" % (grid, name)] = (c4, c4_variant(base, name, grid, with_i64))
    fbs = (r_lo // MIN) * MIN
    nb = (r_hi - fbs) // MIN + 1
    for name in VARIANTS:
        cols = [PushedAggregate(1, cabi.TSKV_PT_I64, ["mean"] + VARIANTS[name]),
                PushedAggregate(2, cabi.TSKV_PT_F64, ["mean"])]
        queries["runs/series/" + name] = (rp, QueryOption(cols, width=MIN, first_bucket_start=fbs, n_buckets=nb, group_by_series=True))
    scans = {n: engine.prepare(p, q) for n, (p, q) in queries.items()}
    counters, results = {}, {}
    for name, s in scans.items():
        s.run()
        c = engine.counters()
        counters[name] = {k: c[k] for k in ("points_decoded", "rows_in_range", "page_read_count", "kernel_launches",
                                            "elapsed_scan_ms", "elapsed_fused_ms")}
        results[name] = s.finalize()
        for _ in range(args.warmup):
            s.enqueue()
            s.sync()
    runs = {name: [] for name in scans}
    for _ in range(args.rounds):  # alternating, so that every variant sees the same machine
        for name, s in scans.items():
            runs[name].append(time_steps(s, args.steps))
    same, mean_check, states = True, {}, {}
    for prefix in ("c4/one_series", "c4/series", "runs/series"):
        a = results[prefix + "/mean"]
        for variant in ("state_i64", "periods_i64"):
            b = results[prefix + "/" + variant]
            for j, name in enumerate(a.names):
                k = b.names.index(name)
                bits = bool((a.values[j] == b.values[k]).all() and (a.validity[j] == b.validity[k]).all())
                x, y = a.values[j].view(np.float64), b.values[k].view(np.float64)
                rel = float(np.nanmax(np.abs(x - y) / np.maximum(np.abs(x), 1e-300))) if x.size else 0.0
                mean_check["%s/%s col %s" % (prefix, variant, name[0])] = {"bit_identical": bits, "max_rel_diff": rel}
                same &= bits or (rel <= 1e-12 and bool((a.validity[j] == b.validity[k]).all()))
        b, p = results[prefix + "/state_i64"], results[prefix + "/periods_i64"]
        n, _ = b.column(1, "state_entries")
        same &= bool((p.column(1, "state_entries")[0] == n).all())
        states[prefix] = {"map_entries": int(n.sum()), "periods": int(p.period_csr[1][0][-1]),
                          "selected_rows": int(counters[prefix + "/state_i64"]["rows_in_range"])}
    states["runs/series"]["state_runs"] = n_runs
    out = {"workload": bench.WORKLOADS["C4"].config(args.series)["workload"], "gpu": bench.gpu_identity(0),
           "run_set": {"series": args.run_series, "rows_per_series": args.run_rows, "mean_run_rows": 100},
           "steps_per_round": args.steps, "rounds": args.rounds, "counters": counters, "state_aggs": states,
           "ms_per_step": {n: {"median": statistics.median(v), "min": min(v), "max": max(v), "runs": v} for n, v in runs.items()},
           "mean_check": mean_check, "mean_ok": same}
    line = json.dumps(out)
    print(line)
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "bench_state_agg.json"), "w") as f:
            f.write(line + "\n")
    for s in scans.values():
        s.close()
    c4.close()
    rp.close()
    engine.close()
    if not same:
        sys.exit(1)


if __name__ == "__main__":
    main()
