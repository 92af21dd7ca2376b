"""The cost of increase on the C4 workload (bench.py) grouped by series, in alternating runs on one GPU:
  mean               C4's query, every column asking for MEAN only
  mean_increase_i64  the same plus increase(time, x) of the i64 column (column 1)
  mean_increase_f64  the same plus increase(time, x) of the f64 column (column 2)
and the same three on a page set with overlap merge groups (`merge_*`, --merge-series series): every series holds a
chunk file of 10 column groups x 1000 rows (10 s apart, an i64 and an f64 column) and a delta chunk file of 3000 rows
over the last 3000 rows of that range, so each series ends in one merge group of 4 chunks and 6000 rows (the merged
rows' increase runs in k_merge_increase, one thread per merge group), GROUP BY series over 1-minute buckets.

  python tools/bench_increase.py [--series N] [--merge-series M] [--steps K] [--warmup W] [--rounds R] [--out DIR]

Prints one JSON line: ms per step of each variant (median, min, max over the rounds; a step is one enqueue of the prepared
scan followed by its sync), the card's name and power limit read in the same process, the counters of each variant
(kernel_launches and elapsed_fused_ms include the increase kernels), and per column whether the MEAN outputs of the
increase variants equal the `mean` variant's (integer columns bit for bit, f64 within 1e-12 relative: its sums are added
with atomics). Exits non-zero otherwise. Writes the JSON to DIR/bench_increase.json."""
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


def with_increases(q, inc_cols):
    """q grouped by series with every column asking for MEAN, and an increase of each column in `inc_cols`."""
    cols = [PushedAggregate(c.column_id, c.phys_type, ["mean"] + (["increase"] if c.column_id in inc_cols else []))
            for c in q.columns]
    return QueryOption(cols, series_ids=q.series_ids, time_ranges=q.time_ranges, origin=q.origin, width=q.width,
                       first_bucket_start=q.first_bucket_start, n_buckets=q.n_buckets, group_by_series=True,
                       predicates=[(c, pt, op, v) for c, pt, op, v in q.predicates])


def merge_arena(n_series):
    """(arena, descs, chunk file of every column group) of the merge variant (see the module docstring)."""
    rng = np.random.default_rng(7)
    b = datagen.ArenaBuilder()
    files = []
    step, t0 = 10_000_000_000, datagen.TSBS_T0
    for sid in range(n_series):
        for k in range(10):
            ts = t0 + (np.arange(1000, dtype=np.int64) + 1000 * k) * step
            b.add_column_group(sid, ts, [(1, cabi.TSKV_PT_I64, np.cumsum(rng.integers(0, 9, 1000)), None),
                                         (2, cabi.TSKV_PT_F64, np.cumsum(rng.random(1000)), None)])
            files.append(1)
        ts = t0 + (np.arange(3000, dtype=np.int64) + 7000) * step
        b.add_column_group(sid, ts, [(1, cabi.TSKV_PT_I64, np.cumsum(rng.integers(0, 9, 3000)), None),
                                     (2, cabi.TSKV_PT_F64, np.cumsum(rng.random(3000)), None)])
        files.append(2)
    a, d = b.finish()
    return a, d, np.asarray(files, dtype=np.uint64), t0, step


def merge_queries(n_series, t0, step):
    w = 60_000_000_000
    fbs = t0 - (t0 % w)
    nb = (t0 + 10_000 * step - fbs) // w + 1
    ids = np.arange(n_series, dtype=np.uint32)

    def q(inc_cols):
        return QueryOption([PushedAggregate(c, pt, ["mean"] + (["increase"] if c in inc_cols else []))
                            for c, pt in ((1, cabi.TSKV_PT_I64), (2, cabi.TSKV_PT_F64))],
                           series_ids=ids, width=w, first_bucket_start=fbs, n_buckets=int(nb), group_by_series=True)
    return {"merge_mean": q(()), "merge_mean_increase_i64": q((1,)), "merge_mean_increase_f64": q((2,))}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--series", type=int, default=bench.WORKLOADS["C4"].default_series)
    ap.add_argument("--merge-series", type=int, default=1000)
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()

    engine = Engine(0)
    g = bench.generate_shard(args.series, 0, 1)
    pages = engine.upload_pages(g.arena, g.descs)
    base = bench.make_query(bench.WORKLOADS["C4"].select(args.series))
    queries = {"mean": with_increases(base, ()), "mean_increase_i64": with_increases(base, (1,)),
               "mean_increase_f64": with_increases(base, (2,))}
    scans = {name: engine.prepare(pages, q) for name, q in queries.items()}
    ma, md, mfiles, mt0, mstep = merge_arena(args.merge_series)
    mpages = engine.upload_pages(ma, md)
    mpages.set_chunk_files(mfiles)
    mqueries = merge_queries(args.merge_series, mt0, mstep)
    scans.update({name: engine.prepare(mpages, q) for name, q in mqueries.items()})
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
    ident = bench.gpu_identity(0)
    same, mean_check = True, {}
    for base_name, other in (("mean", "mean_increase_i64"), ("mean", "mean_increase_f64"),
                             ("merge_mean", "merge_mean_increase_i64"), ("merge_mean", "merge_mean_increase_f64")):
        a, b = results[base_name], results[other]
        for col, pt in ((c.column_id, c.phys_type) for c in base.columns):
            j, k = a.names.index((col, "mean")), b.names.index((col, "mean"))
            bits = bool((a.values[j] == b.values[k]).all() and (a.validity[j] == b.validity[k]).all())
            x, y = a.values[j].view(np.float64), b.values[k].view(np.float64)
            rel = float(np.max(np.abs(x - y) / np.maximum(np.abs(x), 1e-300))) if x.size else 0.0
            mean_check["%s col %d" % (other, col)] = {"bit_identical": bits, "max_rel_diff": rel}
            same &= bits or (pt == cabi.TSKV_PT_F64 and rel <= 1e-12 and bool((a.validity[j] == b.validity[k]).all()))
    increases = {}
    for name, col in (("mean_increase_i64", 1), ("mean_increase_f64", 2), ("merge_mean_increase_i64", 1),
                      ("merge_mean_increase_f64", 2)):
        v, ok = results[name].column(col, "increase")
        increases[name] = {"cells": int(ok.sum()), "first": float(v[ok][0]) if ok.any() else None}
    out = {"workload": bench.WORKLOADS["C4"].config(args.series)["workload"] + " GROUP BY series",
           "merge_workload": "%d series x (10 x 1000 rows + a 3000-row delta file), GROUP BY series" % args.merge_series,
           "gpu": ident,
           "steps_per_round": args.steps, "rounds": args.rounds, "counters": counters, "increases": increases,
           "ms_per_step": {n: {"median": statistics.median(v), "min": min(v), "max": max(v), "runs": v} for n, v in runs.items()},
           "mean_check": mean_check, "mean_ok": same}
    line = json.dumps(out)
    print(line)
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "bench_increase.json"), "w") as f:
            f.write(line + "\n")
    for s in scans.values():
        s.close()
    pages.close()
    mpages.close()
    engine.close()
    if not same:
        sys.exit(1)


if __name__ == "__main__":
    main()
