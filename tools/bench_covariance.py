"""The cost of corr on the C4 workload (bench.py): C4's query with only `mean`, and the same query with the column pair
(first column, second column) added (tskv_query.n_pairs: two more passes that decode both columns' pages row-paired), in
alternating runs on one GPU:
  mean            C4's query, every column asking for MEAN only
  mean_corr       the same plus corr of its first two value columns (C4 gives every series ONE field, i64 or f64, so
                  no column group holds both: this measures the passes' page walk and y lookups, with no paired row)
  mean_corr_self  the same plus corr of the first column with itself (every page of that column decoded row-paired
                  twice more: the decode cost of the pair passes)

  python tools/bench_covariance.py [--series N] [--steps K] [--warmup W] [--rounds R] [--out DIR]

Prints one JSON line: ms per step of each variant (median, min, max over the rounds; a step is one enqueue of the prepared
scan followed by its sync), the card's name and power limit read in the same process, the counters of each variant, and
per column whether the MEAN outputs of both variants are bit-identical. An f64 column's sums are added with atomics whose
order can change from run to run (the JSON shows whether two runs of the `mean` scan itself agree bit for bit), so an
f64 column's MEAN may differ within 1e-12 relative; an integer column's must be bit-identical. Exits non-zero otherwise. Writes the JSON to
DIR/bench_covariance.json."""
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


def with_pairs(q, pairs):
    """q with every column asking for MEAN, and the column pairs `pairs`."""
    cols = [PushedAggregate(c.column_id, c.phys_type, ["mean"]) for c in q.columns]
    return QueryOption(cols, series_ids=q.series_ids, time_ranges=q.time_ranges, origin=q.origin, width=q.width,
                       first_bucket_start=q.first_bucket_start, n_buckets=q.n_buckets, group_by_series=q.group_by_series,
                       predicates=[(c, pt, op, v) for c, pt, op, v in q.predicates], pairs=pairs)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--series", type=int, default=bench.WORKLOADS["C4"].default_series)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--rounds", type=int, default=7)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()

    engine = Engine(0)
    g = bench.generate_shard(args.series, 0, 1)
    pages = engine.upload_pages(g.arena, g.descs)
    base = bench.make_query(bench.WORKLOADS["C4"].select(args.series))
    px, py = base.columns[0], base.columns[1]
    queries = {"mean": with_pairs(base, []), "mean_corr": with_pairs(base, [(px.column_id, px.phys_type, py.column_id, py.phys_type)]),
               "mean_corr_self": with_pairs(base, [(px.column_id, px.phys_type, px.column_id, px.phys_type)])}
    scans = {name: engine.prepare(pages, q) for name, q in queries.items()}
    counters, results = {}, {}
    for name, s in scans.items():
        s.run()
        c = engine.counters()
        counters[name] = {k: c[k] for k in ("points_decoded", "rows_in_range", "page_read_count", "kernel_launches",
                                            "elapsed_fused_ms")}
        results[name] = s.finalize()
        for _ in range(args.warmup):
            s.enqueue()
            s.sync()
    runs = {name: [] for name in scans}
    for _ in range(args.rounds):  # alternating, so that every variant sees the same machine
        for name, s in scans.items():
            runs[name].append(time_steps(s, args.steps))
    ident = bench.gpu_identity(0)
    a, b = results["mean"], results["mean_corr"]
    scans["mean"].run()
    again = scans["mean"].finalize()  # the same scan once more: is its f64 MEAN reproducible at all?
    same, mean_check = True, {}
    for col, pt in ((c.column_id, c.phys_type) for c in base.columns):
        j, k = a.names.index((col, "mean")), b.names.index((col, "mean"))
        bits = bool((a.values[j] == b.values[k]).all() and (a.validity[j] == b.validity[k]).all())
        repeat = bool((a.values[j] == again.values[j]).all())
        x, y = a.values[j].view(np.float64), b.values[k].view(np.float64)
        rel = float(np.max(np.abs(x - y) / np.maximum(np.abs(x), 1e-300))) if x.size else 0.0
        mean_check[col] = {"bit_identical": bits, "repeat_bit_identical": repeat, "max_rel_diff": rel}
        same &= bits or (pt == cabi.TSKV_PT_F64 and rel <= 1e-12 and bool((a.validity[j] == b.validity[k]).all()))
    cr, ok = results["mean_corr_self"].pair(0, "corr")
    out = {"workload": bench.WORKLOADS["C4"].config(args.series)["workload"], "gpu": ident,
           "pair": [px.column_id, py.column_id], "self_corr_cells": int(ok.sum()), "self_corr_median": float(np.median(cr[ok])) if ok.any() else None,
           "steps_per_round": args.steps, "rounds": args.rounds, "counters": counters,
           "ms_per_step": {n: {"median": statistics.median(v), "min": min(v), "max": max(v), "runs": v} for n, v in runs.items()},
           "mean_check": mean_check, "mean_ok": same}
    line = json.dumps(out)
    print(line)
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "bench_covariance.json"), "w") as f:
            f.write(line + "\n")
    for s in scans.values():
        s.close()
    pages.close()
    engine.close()
    if not same:
        sys.exit(1)


if __name__ == "__main__":
    main()
