"""The cost of gauge_agg(time, x) on the C4 workload (bench.py), in alternating runs on one GPU. For each grid
(ungrouped, GROUP BY series, and a 5 min / 1 min sliding window, ungrouped) three variants:
  mean          C4's query, every column asking for MEAN only
  gauge_i64     the same plus gauge_agg(time, x) of the i64 column (column 1)
  gauge_f64     the same plus gauge_agg(time, x) of the f64 column (column 2)

  python tools/bench_gauge.py [--series N] [--steps K] [--warmup W] [--rounds R] [--out DIR]

Prints one JSON line: ms per step of each variant (median, min, max over the rounds; a step is one enqueue of the prepared
scan followed by its sync), the card's name and power limit read in the same process, the counters of each variant, the
device time of the gauge passes split by kernel family (records: k_gauge_scan / k_gauge_merge_rows; sort: CUB's radix
sort; reduce: CUB's reduce by key; rest: gather, scatter, fold, check), taken with torch.profiler in a separate pass
after the timed rounds, and whether the MEAN outputs of the gauge variants equal the `mean` variant's (integers bit for
bit, f64 within 1e-12 relative). Exits non-zero otherwise. Writes the JSON to DIR/bench_gauge.json."""
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
from cnosdb_b200.engine import Engine, PushedAggregate, QueryOption, sliding_window_grid  # noqa: E402

MIN = 60_000_000_000


def variant(q, gauge_col, grid):
    cols = [PushedAggregate(c.column_id, c.phys_type, ["mean"] + (["gauge_agg"] if c.column_id == gauge_col else []))
            for c in q.columns]
    kw = dict(series_ids=q.series_ids, time_ranges=q.time_ranges, origin=q.origin, width=q.width,
              first_bucket_start=q.first_bucket_start, n_buckets=q.n_buckets,
              predicates=[(c, pt, op, v) for c, pt, op, v in q.predicates])
    if grid == "ungrouped":
        kw.update(width=0, origin=0, first_bucket_start=0, n_buckets=1)
    elif grid == "series":
        kw.update(group_by_series=True)
    else:  # sliding 5 min / 1 min over the span of C4's tumbling grid
        lo, hi = q.first_bucket_start, q.first_bucket_start + q.n_buckets * q.width - 1
        fbs, nb = sliding_window_grid(lo, hi, 5 * MIN, MIN, 0)
        kw.update(width=5 * MIN, origin=0, first_bucket_start=fbs, n_buckets=nb)
    return QueryOption(cols, **kw)


def family(name):
    n = name.lower()
    if "k_gauge_scan" in n or "k_gauge_merge_rows" in n:
        return "records"
    if "radixsort" in n or "radix_sort" in n:
        return "sort"
    if "reducebykey" in n or "compactinit" in n:
        return "reduce"
    if "gauge" in n:
        return "rest"
    return None


def profile_split(s, steps):
    """{family: device ms per step} of one prepared gauge scan, from torch.profiler's CUDA kernel events."""
    import torch
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(steps):
            s.enqueue()
            s.sync()
        torch.cuda.synchronize()
    out = {"records": 0.0, "sort": 0.0, "reduce": 0.0, "rest": 0.0}
    for e in prof.key_averages():
        f = family(e.key)
        if f:
            out[f] += getattr(e, "device_time_total", getattr(e, "cuda_time_total", 0.0)) / 1000.0 / steps
    return out


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
    queries, slides = {}, {}
    for grid in ("ungrouped", "series", "sliding"):
        for name, col in (("mean", None), ("gauge_i64", 1), ("gauge_f64", 2)):
            queries["%s/%s" % (grid, name)] = variant(base, col, grid)
            slides["%s/%s" % (grid, name)] = MIN if grid == "sliding" else None
    scans = {n: engine.prepare(pages, q, slide=slides[n]) for n, q in queries.items()}
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
    split = {n: profile_split(s, args.steps) for n, s in scans.items() if "gauge" in n}
    ident = bench.gpu_identity(0)
    same, mean_check, gauges = True, {}, {}
    for grid in ("ungrouped", "series", "sliding"):
        a = results[grid + "/mean"]
        for other, col in (("gauge_i64", 1), ("gauge_f64", 2)):
            b = results["%s/%s" % (grid, other)]
            for c in base.columns:
                j, k = a.names.index((c.column_id, "mean")), b.names.index((c.column_id, "mean"))
                bits = bool((a.values[j] == b.values[k]).all() and (a.validity[j] == b.validity[k]).all())
                x, y = a.values[j].view(np.float64), b.values[k].view(np.float64)
                rel = float(np.nanmax(np.abs(x - y) / np.maximum(np.abs(x), 1e-300))) if x.size else 0.0
                mean_check["%s/%s col %d" % (grid, other, c.column_id)] = {"bit_identical": bits, "max_rel_diff": rel}
                same &= bits or (rel <= 1e-12 and bool((a.validity[j] == b.validity[k]).all()))
            n, ok = b.gauge(col, "n")
            gauges["%s/%s" % (grid, other)] = {"cells": int((n > 0).sum()), "points": int(n.sum())}
    out = {"workload": bench.WORKLOADS["C4"].config(args.series)["workload"], "gpu": ident,
           "steps_per_round": args.steps, "rounds": args.rounds, "counters": counters, "gauges": gauges,
           "gauge_ms_per_step_by_family": split,
           "ms_per_step": {n: {"median": statistics.median(v), "min": min(v), "max": max(v), "runs": v} for n, v in runs.items()},
           "mean_check": mean_check, "mean_ok": same}
    line = json.dumps(out)
    print(line)
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "bench_gauge.json"), "w") as f:
            f.write(line + "\n")
    for s in scans.values():
        s.close()
    pages.close()
    engine.close()
    if not same:
        sys.exit(1)


if __name__ == "__main__":
    main()
