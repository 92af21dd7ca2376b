"""The cost of mode(x) and COUNT(DISTINCT x) on the C4 workload (bench.py), in alternating runs on one GPU, ungrouped (C4's
own grid) and grouped by series (`series_*`):
  mean                 C4's query, every column asking for MEAN only
  mode_i64             the same plus mode of the i64 column (column 1)
  mode_f64             the same plus mode of the f64 column (column 2)
  distinct_i64         the same plus COUNT(DISTINCT) of column 1
  mode_distinct_i64    the same plus mode and COUNT(DISTINCT) of column 1 (one gather and one sort serve both)

  python tools/bench_mode.py [--series N] [--steps K] [--warmup W] [--rounds R] [--out DIR]

Prints one JSON line: ms per step of each variant (median, min, max over the rounds; a step is one enqueue of the prepared
scan followed by its sync), the card's name and power limit read in the same process, the counters of each variant, and
whether the MEAN outputs of every variant equal the `mean` variant's (integer columns bit for bit, f64 within 1e-12
relative: its sums are added with atomics). Exits non-zero otherwise. Writes the JSON to DIR/bench_mode.json."""
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

VARIANTS = {"mean": {}, "mode_i64": {1: ["mode"]}, "mode_f64": {2: ["mode"]}, "distinct_i64": {1: ["count_distinct"]},
            "mode_distinct_i64": {1: ["mode", "count_distinct"]}}


def variant(q, extra, by_series):
    """q with every column asking for MEAN, plus the aggregates of `extra` (column id -> names)."""
    cols = [PushedAggregate(c.column_id, c.phys_type, ["mean"] + extra.get(c.column_id, [])) for c in q.columns]
    return QueryOption(cols, series_ids=q.series_ids, time_ranges=q.time_ranges, origin=q.origin, width=q.width,
                       first_bucket_start=q.first_bucket_start, n_buckets=q.n_buckets, group_by_series=by_series,
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
    queries = {}
    for by_series in (False, True):
        for name, extra in VARIANTS.items():
            queries[("series_" if by_series else "") + name] = variant(base, extra, by_series)
    scans = {name: engine.prepare(pages, q) for name, q in queries.items()}
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
    for name in scans:
        a = results["series_mean" if name.startswith("series_") else "mean"]
        b = results[name]
        for col, pt in ((c.column_id, c.phys_type) for c in base.columns):
            j, k = a.names.index((col, "mean")), b.names.index((col, "mean"))
            bits = bool((a.values[j] == b.values[k]).all() and (a.validity[j] == b.validity[k]).all())
            x, y = a.values[j].view(np.float64), b.values[k].view(np.float64)
            rel = float(np.nanmax(np.abs(x - y) / np.maximum(np.abs(x), 1e-300))) if x.size else 0.0
            mean_check["%s col %d" % (name, col)] = {"bit_identical": bits, "max_rel_diff": rel}
            same &= bits or (pt == cabi.TSKV_PT_F64 and rel <= 1e-12 and bool((a.validity[j] == b.validity[k]).all()))
    out = {"workload": bench.WORKLOADS["C4"].config(args.series)["workload"], "gpu": ident,
           "steps_per_round": args.steps, "rounds": args.rounds, "counters": counters,
           "ms_per_step": {n: {"median": statistics.median(v), "min": min(v), "max": max(v), "runs": v} for n, v in runs.items()},
           "mean_check": mean_check, "mean_ok": same}
    line = json.dumps(out)
    print(line)
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "bench_mode.json"), "w") as f:
            f.write(line + "\n")
    for s in scans.values():
        s.close()
    pages.close()
    engine.close()
    if not same:
        sys.exit(1)


if __name__ == "__main__":
    main()
