"""Labelled time buckets against the tumbling and edge scans on the C4 workload (bench.py), in alternating runs on one GPU:
  tumbling_1min    the C4 query (tumbling 1-minute buckets, tskvgpu_scan_prepare)
  edges_1min       the same 1-minute grid handed in as edges (tskvgpu_scan_prepare_edges)
  minute_of_hour   the same 1-minute edges labelled with their minute of the hour (tskvgpu_scan_prepare_labels):
                   GROUP BY date_part('minute', time), ~168 edge buckets into 60 cells

  python tools/bench_bucket_labels.py [--series N] [--steps K] [--warmup W] [--rounds R] [--out DIR]

Prints one JSON line: ms per step of each variant (median, min, max over the rounds; a step is one enqueue of the
prepared scan followed by its sync), the card's name and power limit read in the same process, the counters of each
variant, and whether minute_of_hour equals the host fold of edges_1min by minute of the hour (counts, integer sums,
min / max and the integer mean bit for bit; f64 sums and means within 1e-9 relative: the order of the additions
differs). Exits non-zero if not. Writes the JSON to DIR/bench_bucket_labels.json."""
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
from bench_bucket_edges import edge_query, time_steps, uniform_edges  # noqa: E402
from cnosdb_b200 import cabi  # noqa: E402
from cnosdb_b200.engine import Engine  # noqa: E402

MINUTE = 60 * 10**9


def minute_labels(edges):
    """Minute of the hour of every 1-minute edge bucket (UTC; floor before 1970)."""
    return (edges[:-1] // MINUTE % 60).astype(np.uint32)


def fold_equals(labelled, fine, labels):
    """Does the labelled result equal the edge scan's result folded by label? (one group: GROUP BY bucket)"""
    n_out = labelled.n_buckets
    for col in sorted({c for c, _ in labelled.names}):
        pt = labelled.phys[col]
        cnt, cok = fine.column(col, "count")
        s, sok = fine.column(col, "sum")
        cnt, s, sok = cnt[0], s[0], sok[0]
        fold_cnt = np.bincount(labels, weights=cnt.astype(np.float64), minlength=n_out).astype(np.uint64)
        if pt == cabi.TSKV_PT_F64:
            fold_sum = np.bincount(labels, weights=np.where(sok, s, 0.0), minlength=n_out)
        else:
            fold_sum = np.zeros(n_out, dtype=s.dtype)
            with np.errstate(over="ignore"):
                np.add.at(fold_sum, labels, np.where(sok, s, 0).astype(s.dtype))
        for agg in ("count", "sum", "min", "max", "mean"):
            g, gok = labelled.column(col, agg)
            g, gok = g[0], gok[0]
            if agg == "count":
                if not (g == fold_cnt).all():
                    return False
                continue
            have = fold_cnt > 0
            if not (gok == have).all():
                return False
            if agg in ("min", "max"):
                v, ok = fine.column(col, agg)
                v, ok = v[0], ok[0]
                exp = np.array([(v[ok & (labels == j)].min() if agg == "min" else v[ok & (labels == j)].max())
                                if have[j] else 0 for j in range(n_out)], dtype=v.dtype)
                if not (g[have] == exp[have]).all():
                    return False
                continue
            exp = fold_sum if agg == "sum" else fold_sum.astype(np.float64) / np.maximum(fold_cnt, 1).astype(np.float64)
            if pt == cabi.TSKV_PT_F64:
                if not (np.abs(g[have] - exp[have]) <= 1e-9 * np.maximum(np.abs(exp[have]), 1e-300)).all():
                    return False
            elif not (g[have] == exp[have]).all():
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
    e = uniform_edges(tumbling)
    lab = minute_labels(e)
    labelled = edge_query(tumbling, e)
    labelled.n_buckets = 60
    scans = {"tumbling_1min": engine.prepare(pages, tumbling),
             "edges_1min": engine.prepare(pages, edge_query(tumbling, e), edges=e),
             "minute_of_hour": engine.prepare(pages, labelled, edges=e, labels=lab)}
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
    same = fold_equals(results["minute_of_hour"], results["edges_1min"], lab)
    out = {"workload": bench.WORKLOADS["C4"].config(args.series)["workload"], "gpu": ident,
           "buckets": {"tumbling_1min": tumbling.n_buckets, "edges_1min": len(e) - 1,
                       "minute_of_hour": {"edge_buckets": len(e) - 1, "cells": 60}},
           "steps_per_round": args.steps, "rounds": args.rounds, "counters": counters,
           "ms_per_step": {n: {"median": statistics.median(v), "min": min(v), "max": max(v), "runs": v} for n, v in runs.items()},
           "minute_of_hour_equals_folded_edges": same}
    line = json.dumps(out)
    print(line)
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "bench_bucket_labels.json"), "w") as f:
            f.write(line + "\n")
    for s in scans.values():
        s.close()
    pages.close()
    engine.close()
    if not same:
        sys.exit(1)


if __name__ == "__main__":
    main()
