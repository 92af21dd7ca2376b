"""GROUP BY tags on the C4 workload (bench.py): the C4 query with its selected series mapped to G groups by a hash of the
series id (so a group's members are scattered through the arena, as tag values are), against the ungrouped scan and
GROUP BY series, in alternating rounds on one GPU.

  python tools/bench_group_by_tag.py [--series N] [--steps K] [--warmup W] [--rounds R] [--out DIR]

Variants: ungrouped, G = 1, 10, 1000, one group per selected series, group_by_series. Prints one JSON line: ms per step
of each variant (median, min, max over the rounds; a step is one enqueue of the prepared scan followed by its sync), the
card's name and power limit read in the same process, and whether a sample of groups (three of G = 10, three of G = 1000)
equals the ungrouped scans of their members (integer outputs exact, f64 sums / means within 1e-12 relative). Writes the
JSON to DIR/bench_group_by_tag.json."""
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
from cnosdb_b200.engine import Engine  # noqa: E402


def hash_groups(series_ids, n_groups):
    """Group of every selected series: a multiplicative hash of its id, mod n_groups."""
    h = (np.asarray(series_ids, dtype=np.uint64) * np.uint64(2654435761)) & np.uint64(0xFFFFFFFF)
    return (h % np.uint64(n_groups)).astype(np.uint32)


def time_steps(scan, steps):
    t0 = time.perf_counter()
    for _ in range(steps):
        scan.enqueue()
        scan.sync()
    return (time.perf_counter() - t0) * 1e3 / steps


def check_sample(engine, pages, q, sel, gmap, n_groups, groups):
    """The grouped cells of `groups` == the ungrouped scans of their members."""
    from tests.test_gpu_group_by_tag import assert_cells_equal, with_series
    got = engine.scan_aggregate(pages, q, group_ids=gmap, n_groups=n_groups)
    nb = q.n_buckets
    try:
        for g in groups:
            sub = engine.scan_aggregate(pages, with_series(q, sel[gmap == g]))
            cells = slice(g * nb, (g + 1) * nb)
            for j, (col, agg) in enumerate(got.names):
                assert_cells_equal(got.values[j][cells], got.validity[j][cells], sub.values[j], sub.validity[j], got, col, agg,
                                   "C4 G=%d group %d" % (n_groups, g))
        return True
    except AssertionError as e:
        print("sample check failed: %s" % e, file=sys.stderr)
        return False


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
    sel = np.asarray(bench.WORKLOADS["C4"].select(args.series), dtype=np.uint32)
    q = bench.make_query(sel)
    by_series = bench.make_query(sel)
    by_series.group_by_series = True
    maps = {n: hash_groups(sel, n) for n in (1, 10, 1000)}
    scans = {"ungrouped": engine.prepare(pages, q)}
    for n, m in maps.items():
        scans["G=%d" % n] = engine.prepare(pages, q, group_ids=m, n_groups=n)
    scans["G=per_series"] = engine.prepare(pages, q, group_ids=np.arange(len(sel), dtype=np.uint32), n_groups=len(sel))
    scans["group_by_series"] = engine.prepare(pages, by_series)
    for s in scans.values():
        s.run()
        for _ in range(args.warmup):
            s.enqueue()
            s.sync()
    runs = {name: [] for name in scans}
    for _ in range(args.rounds):  # alternating, so that every variant sees the same machine
        for name, s in scans.items():
            runs[name].append(time_steps(s, args.steps))
    ident = bench.gpu_identity(0)
    ok = check_sample(engine, pages, q, sel, maps[10], 10, (0, 4, 9)) and check_sample(engine, pages, q, sel, maps[1000], 1000, (0, 500, 999))
    ms = {n: {"median": statistics.median(v), "min": min(v), "max": max(v), "runs": v} for n, v in runs.items()}
    base = ms["ungrouped"]["median"]
    out = {"workload": bench.WORKLOADS["C4"].config(args.series)["workload"], "gpu": ident, "selected_series": int(len(sel)),
           "buckets": q.n_buckets, "steps_per_round": args.steps, "rounds": args.rounds, "ms_per_step": ms,
           "median_vs_ungrouped": {n: v["median"] / base for n, v in ms.items()}, "sample_check_ok": ok}
    line = json.dumps(out)
    print(line)
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "bench_group_by_tag.json"), "w") as f:
            f.write(line + "\n")
    for s in scans.values():
        s.close()
    pages.close()
    engine.close()
    if not ok:
        sys.exit(1)


if __name__ == "__main__":
    main()
