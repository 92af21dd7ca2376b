"""Explicit time-bucket edges against the tumbling scan on the C4 workload (bench.py), in alternating runs on one GPU:
  tumbling_1min    the C4 query (tumbling 1-minute buckets, tskvgpu_scan_prepare)
  edges_1min       the same 1-minute grid handed in as edges (tskvgpu_scan_prepare_edges)
  edges_50s_70s    irregular edges over the same span: buckets alternating 50 s and 70 s

  python tools/bench_bucket_edges.py [--series N] [--steps K] [--warmup W] [--rounds R] [--out DIR]

Prints one JSON line: ms per step of each variant (median, min, max over the rounds; a step is one enqueue of the
prepared scan followed by its sync), the card's name and power limit read in the same process, the counters of each
variant, and whether the two 1-minute variants give equal outputs (counts, integer sums, min / max bit for bit; f64 sums
and means within 1e-12 relative). With TSKV_DEBUG_BINS=1 TSKV_NO_GRAPH=1 the library prints each bin's kernel time.
Writes the JSON to DIR/bench_bucket_edges.json."""
import argparse
import copy
import json
import os
import statistics
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import bench  # noqa: E402
from cnosdb_b200 import cabi  # noqa: E402
from cnosdb_b200.engine import Engine  # noqa: E402


def edge_query(tumbling, edges):
    q = copy.copy(tumbling)
    q.width, q.origin, q.first_bucket_start, q.n_buckets = 0, 0, 0, len(edges) - 1
    q._keep = None
    return q


def uniform_edges(q):
    return q.first_bucket_start + np.arange(q.n_buckets + 1, dtype=np.int64) * q.width


def irregular_edges(q, a=50 * 10**9, b=70 * 10**9):
    """Buckets alternating a and b wide from the grid's start past its end."""
    lo, hi = q.first_bucket_start, q.first_bucket_start + q.n_buckets * q.width
    out = [lo]
    while out[-1] < hi:
        out.append(out[-1] + (a if len(out) % 2 else b))
    return np.array(out, dtype=np.int64)


def time_steps(scan, steps):
    t0 = time.perf_counter()
    for _ in range(steps):
        scan.enqueue()
        scan.sync()
    return (time.perf_counter() - t0) * 1e3 / steps


def outputs_equal(a, b):
    for j, (col, agg) in enumerate(a.names):
        if not (a.validity[j] == b.validity[j]).all():
            return False
        ok = a.validity[j]
        if agg in ("sum", "mean") and a.phys[col] == cabi.TSKV_PT_F64:
            x, y = a.values[j][ok].view(np.float64), b.values[j][ok].view(np.float64)
            if not (np.abs(x - y) <= 1e-12 * np.maximum(np.abs(y), 1e-300)).all():
                return False
        elif not (a.values[j][ok] == b.values[j][ok]).all():
            return False
    return True


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
    sel = bench.WORKLOADS["C4"].select(args.series)
    tumbling = bench.make_query(sel)
    e_uni, e_irr = uniform_edges(tumbling), irregular_edges(tumbling)
    scans = {"tumbling_1min": engine.prepare(pages, tumbling),
             "edges_1min": engine.prepare(pages, edge_query(tumbling, e_uni), edges=e_uni),
             "edges_50s_70s": engine.prepare(pages, edge_query(tumbling, e_irr), edges=e_irr)}
    counters, results = {}, {}
    for name, s in scans.items():
        s.run()
        c = engine.counters()
        counters[name] = {k: c[k] for k in ("points_decoded", "rows_in_range", "page_read_count")}
        results[name] = s.finalize()
        for _ in range(args.warmup):
            s.enqueue()
            s.sync()
    runs = {name: [] for name in scans}
    for _ in range(args.rounds):  # alternating, so that every variant sees the same machine
        for name, s in scans.items():
            runs[name].append(time_steps(s, args.steps))
    ident = bench.gpu_identity(0)
    same = outputs_equal(results["edges_1min"], results["tumbling_1min"])
    out = {"workload": bench.WORKLOADS["C4"].config(args.series)["workload"], "gpu": ident,
           "buckets": {"tumbling_1min": tumbling.n_buckets, "edges_1min": len(e_uni) - 1, "edges_50s_70s": len(e_irr) - 1},
           "steps_per_round": args.steps, "rounds": args.rounds, "counters": counters,
           "ms_per_step": {n: {"median": statistics.median(v), "min": min(v), "max": max(v), "runs": v} for n, v in runs.items()},
           "edges_1min_equals_tumbling": same}
    line = json.dumps(out)
    print(line)
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "bench_bucket_edges.json"), "w") as f:
            f.write(line + "\n")
    for s in scans.values():
        s.close()
    pages.close()
    engine.close()
    if not same:
        sys.exit(1)


if __name__ == "__main__":
    main()
