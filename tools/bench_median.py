"""The cost of median on the C4 workload (bench.py), in alternating runs on one GPU:
  mean             C4's query, every column asking for MEAN only
  mean_median_i64  the same plus the median of the i64 column (column 1)
  mean_median_f64  the same plus the median of the f64 column (column 2)
  tags_median_f64  the same as mean_median_f64 grouped by tags: 1000 groups (series slot % 1000), under the median
                   cell cap (1000 x the buckets)

  python tools/bench_median.py [--series N] [--steps K] [--warmup W] [--rounds R] [--out DIR]

Prints one JSON line: ms per step of each variant (median, min, max over the rounds; a step is one enqueue of the prepared
scan followed by its sync), the card's name and power limit read in the same process, the counters of each variant
(kernel_launches and elapsed_fused_ms include the 8 selection passes), and per column whether the MEAN outputs of the median variants equal the `mean`
variant's (integer columns bit for bit, f64 within 1e-12 relative: its sums are added with atomics). Exits non-zero
otherwise. Writes the JSON to DIR/bench_median.json."""
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
from cnosdb_b200 import cabi  # noqa: E402
from cnosdb_b200.engine import Engine, PushedAggregate, QueryOption  # noqa: E402


def with_medians(q, median_cols):
    """q with every column asking for MEAN, and a median of each column in `median_cols`."""
    cols = [PushedAggregate(c.column_id, c.phys_type, ["mean"] + (["median"] if c.column_id in median_cols else []))
            for c in q.columns]
    return QueryOption(cols, series_ids=q.series_ids, time_ranges=q.time_ranges, origin=q.origin, width=q.width,
                       first_bucket_start=q.first_bucket_start, n_buckets=q.n_buckets, group_by_series=q.group_by_series,
                       predicates=[(c, pt, op, v) for c, pt, op, v in q.predicates])


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--series", type=int, default=bench.WORKLOADS["C4"].default_series)
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()

    engine = Engine(0)
    g = bench.generate_shard(args.series, 0, 1)
    pages = engine.upload_pages(g.arena, g.descs)
    base = bench.make_query(bench.WORKLOADS["C4"].select(args.series))
    n_sel = len(base.series_ids) if base.series_ids is not None else args.series
    gids = (np.arange(n_sel) % 1000).astype(np.uint32)
    queries = {"mean": (with_medians(base, ()), {}), "mean_median_i64": (with_medians(base, (1,)), {}),
               "mean_median_f64": (with_medians(base, (2,)), {}),
               "tags_median_f64": (with_medians(base, (2,)), {"group_ids": gids, "n_groups": 1000})}
    scans = {name: engine.prepare(pages, q, **kw) for name, (q, kw) in queries.items()}
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
    a = results["mean"]
    same, mean_check = True, {}
    for other in ("mean_median_i64", "mean_median_f64"):
        b = results[other]
        for col, pt in ((c.column_id, c.phys_type) for c in base.columns):
            j, k = a.names.index((col, "mean")), b.names.index((col, "mean"))
            bits = bool((a.values[j] == b.values[k]).all() and (a.validity[j] == b.validity[k]).all())
            x, y = a.values[j].view(np.float64), b.values[k].view(np.float64)
            rel = float(np.max(np.abs(x - y) / np.maximum(np.abs(x), 1e-300))) if x.size else 0.0
            mean_check["%s col %d" % (other, col)] = {"bit_identical": bits, "max_rel_diff": rel}
            same &= bits or (pt == cabi.TSKV_PT_F64 and rel <= 1e-12 and bool((a.validity[j] == b.validity[k]).all()))
    medians = {}
    for name, col in (("mean_median_i64", 1), ("mean_median_f64", 2), ("tags_median_f64", 2)):
        v, ok = results[name].column(col, "median")
        medians[name] = {"cells": int(ok.sum()), "first": float(v[ok][0]) if ok.any() else None}
    out = {"workload": bench.WORKLOADS["C4"].config(args.series)["workload"], "gpu": ident,
           "steps_per_round": args.steps, "rounds": args.rounds, "counters": counters, "medians": medians,
           "ms_per_step": {n: {"median": statistics.median(v), "min": min(v), "max": max(v), "runs": v} for n, v in runs.items()},
           "mean_check": mean_check, "mean_ok": same}
    line = json.dumps(out)
    print(line)
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "bench_median.json"), "w") as f:
            f.write(line + "\n")
    for s in scans.values():
        s.close()
    pages.close()
    engine.close()
    if not same:
        sys.exit(1)


if __name__ == "__main__":
    main()
