"""Sliding windows against the tumbling scan on the C4 workload (bench.py): time_window(time, 5 min, 1 min) over the
selected series against the tumbling 1-minute scan of the same selection, in alternating runs on one GPU.

  python tools/bench_sliding.py [--series N] [--steps K] [--warmup W] [--rounds R] [--check-series S] [--out DIR]

Prints one JSON line: ms per step of each variant (median, min, max over the rounds; a step is one enqueue of the
prepared scan followed by its sync), the card's name and power limit read in the same process, and whether the sliding
result equals the oracle's tumbling 1-minute panes folded into windows on a sample of the selected series (counts,
integer sums, min / max exact; f64 sums / means within 1e-12 relative). Writes the JSON to DIR/bench_sliding.json."""
import argparse
import json
import os
import statistics
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import bench  # noqa: E402
from cnosdb_b200.engine import Engine, sliding_window_grid  # noqa: E402

WINDOW, SLIDE = 5 * bench.W_NS, bench.W_NS


def sliding_query(tumbling):
    """The C4 query with 5-minute windows every minute over the span the tumbling grid covers."""
    lo = tumbling.first_bucket_start
    hi = lo + tumbling.n_buckets * tumbling.width - 1
    fbs, nb = sliding_window_grid(lo, hi, WINDOW, SLIDE)
    return bench.QueryOption(tumbling.columns, series_ids=tumbling.series_ids, width=WINDOW, first_bucket_start=fbs,
                             n_buckets=nb)


def time_steps(scan, steps):
    t0 = time.perf_counter()
    for _ in range(steps):
        scan.enqueue()
        scan.sync()
    return (time.perf_counter() - t0) * 1e3 / steps


def check_sample(engine, pages, g, sel, n_check):
    """GPU sliding windows of a sample of the selection == the oracle's tumbling 1-minute panes, folded."""
    from oracle import pyoracle as orc
    from tests.test_gpu_sliding_window import _pane_query, assert_folded, fold_panes
    sample = np.sort(np.random.default_rng(1).choice(sel, size=min(n_check, len(sel)), replace=False)).astype(np.uint32)
    q = sliding_query(bench.make_query(sample))
    k = -(-WINDOW // SLIDE)
    got = engine.scan_aggregate(pages, q, slide=SLIDE)
    panes = orc.scan_aggregate(g.arena, g.descs, _pane_query(q, SLIDE, k), n_threads=os.cpu_count() or 1)
    try:
        assert_folded(got, fold_panes(panes, k, q.n_buckets), "C4 sample")
        return True, int(len(sample))
    except AssertionError as e:
        print("sample check failed: %s" % e, file=sys.stderr)
        return False, int(len(sample))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--series", type=int, default=bench.WORKLOADS["C4"].default_series)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--rounds", type=int, default=7)
    ap.add_argument("--check-series", type=int, default=2000)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()

    engine = Engine(0)
    g = bench.generate_shard(args.series, 0, 1)
    pages = engine.upload_pages(g.arena, g.descs)
    sel = bench.WORKLOADS["C4"].select(args.series)
    tumbling = bench.make_query(sel)
    sliding = sliding_query(tumbling)
    scans = {"tumbling_1min": engine.prepare(pages, tumbling), "sliding_5min_by_1min": engine.prepare(pages, sliding, slide=SLIDE)}
    points = {}
    for name, s in scans.items():
        s.run()
        points[name] = engine.counters()["points_decoded"]
        for _ in range(args.warmup):
            s.enqueue()
            s.sync()
    runs = {name: [] for name in scans}
    for _ in range(args.rounds):  # alternating, so that both variants see the same machine
        for name, s in scans.items():
            runs[name].append(time_steps(s, args.steps))
    ident = bench.gpu_identity(0)
    ok, n_checked = check_sample(engine, pages, g, sel, args.check_series)
    out = {"workload": bench.WORKLOADS["C4"].config(args.series)["workload"], "gpu": ident,
           "window_ns": WINDOW, "slide_ns": SLIDE, "windows": sliding.n_buckets, "tumbling_buckets": tumbling.n_buckets,
           "steps_per_round": args.steps, "rounds": args.rounds, "points_decoded": points,
           "ms_per_step": {n: {"median": statistics.median(v), "min": min(v), "max": max(v), "runs": v} for n, v in runs.items()},
           "oracle_sample_series": n_checked, "oracle_sample_ok": ok}
    out["sliding_minus_tumbling_ms"] = out["ms_per_step"]["sliding_5min_by_1min"]["median"] - out["ms_per_step"]["tumbling_1min"]["median"]
    line = json.dumps(out)
    print(line)
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "bench_sliding.json"), "w") as f:
            f.write(line + "\n")
    for s in scans.values():
        s.close()
    pages.close()
    engine.close()
    if not ok:
        sys.exit(1)


if __name__ == "__main__":
    main()
