"""Scan prologue (series selection, work list, state init) across series / column-group shapes, with and without a
selection list and a field predicate, on one GPU. Every scan runs un-captured (TSKV_NO_GRAPH=1) so that its events
time each pass.

  python tools/bench_worklist_shapes.py [--shapes a,b] [--steps K] [--warmup W] [--out DIR]
  python tools/bench_worklist_shapes.py --compare DIR_A DIR_B

Shapes (C4's generator: mixed i64 / f64 pages, 20 % jittered timestamps; the column groups of a series are C4 series
relabelled into one series, so they share their time span):
  4x2000     4 series x 2000 column groups of 1000 rows
  1000x100   1000 series x 100 column groups of 1000 rows
  100000x40  100 000 series x 40 column groups of 100 rows
  skewed     one series of 1000 column groups among 99 000 single-group series (1000 rows each)
  C4         bench.py's C4 page set (1 000 000 series, one column group each)
Variants: all series / every 10th series (every 2nd below 10 series), each without and with the predicate
column 1 > 0. The C4 query (count, sum, min, max, mean of columns 1 and 2 per 1-minute bucket) throughout.

Prints one JSON line per shape and writes them, with the outputs of every scan (DIR/<shape>-<variant>.npz), to DIR:
median / min / max over the steps of elapsed_scan_ms and of elapsed_scan_ms - elapsed_fused_ms (the prologue plus the
epilogue: export and finalize of the cells, the same in both builds of one comparison), the reader counters, and the
card's name and power limit. --compare checks two such directories against each other: counters equal, integer
outputs equal, f64 sums / means within 1e-12 relative."""
import argparse
import json
import os
import statistics
import sys
import tempfile

import numpy as np

os.environ["TSKV_NO_GRAPH"] = "1"
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import bench  # noqa: E402
from cnosdb_b200 import cabi, datagen  # noqa: E402

# generated series, column groups per series (None: skewed), rows per column group
SHAPES = {"4x2000": (8000, 2000, 1000), "1000x100": (100_000, 100, 1000), "100000x40": (4_000_000, 40, 100),
          "skewed": (100_000, None, 1000), "C4": (1_000_000, 1, 1000)}
PRED = [(1, cabi.TSKV_PT_I64, ">", 0)]
COUNTERS = ("page_read_count", "page_read_bytes", "pruned_page_count", "points_decoded")


def build_shape(name):
    """(generated set, descriptor table with the shape's series ids)."""
    n_raw, groups, n_points = SHAPES[name]
    g = datagen.generate(n_raw, series_stride=1, n_points=n_points, **bench.WORKLOADS["C4"].gen_kw)
    d = g.descs.copy()
    sid = d["series_id"].astype(np.int64)
    if name == "skewed":
        d["series_id"] = np.where(sid < 1000, 0, sid - 999)
    else:
        d["series_id"] = sid // groups
    return g, d


def run_variant(engine, pages, q, steps, warmup):
    scan = engine.prepare(pages, q)
    for _ in range(warmup):
        scan.enqueue()
        scan.sync()
    total, rest = [], []
    for _ in range(steps):
        scan.enqueue()
        scan.sync()
        c = engine.counters()
        total.append(c["elapsed_scan_ms"])
        rest.append(c["elapsed_scan_ms"] - c["elapsed_fused_ms"])
    counters = {k: int(c[k]) for k in COUNTERS}
    res = scan.finalize()
    scan.close()
    stat = lambda xs: {"median": statistics.median(xs), "min": min(xs), "max": max(xs)}  # noqa: E731
    return {"scan_ms": stat(total), "prologue_epilogue_ms": stat(rest), "counters": counters}, res


def measure(args):
    from cnosdb_b200.engine import Engine
    os.makedirs(args.out, exist_ok=True)
    engine = Engine(0)
    card = bench.gpu_identity(0)
    lines = []
    for name in args.shapes.split(","):
        g, descs = build_shape(name)
        pages = engine.upload_pages(g.arena, descs)
        ids = np.unique(descs["series_id"]).astype(np.uint32)
        subset = ids[::10] if len(ids) >= 10 else ids[::2]
        out = {"shape": name, "series": int(len(ids)), "field_pages": int((descs["phys_type"] != cabi.TSKV_PT_TIME).sum()),
               "card": card, "steps": args.steps, "variants": {}}
        for sel_name, sel in (("all", None), ("subset", subset)):
            for pred_name, pred in (("", []), ("+pred", PRED)):
                variant = sel_name + pred_name
                r, res = run_variant(engine, pages, bench.WORKLOADS["C4"].query(sel, predicates=pred), args.steps, args.warmup)
                out["variants"][variant] = r
                is_float = np.array([agg == "mean" or (agg == "sum" and res.phys[col] == cabi.TSKV_PT_F64) for col, agg in res.names])
                np.savez(os.path.join(args.out, "%s-%s.npz" % (name, variant)), values=res.values, validity=res.validity,
                         is_float=is_float, counters=np.array([r["counters"][k] for k in COUNTERS], dtype=np.int64))
        pages.close()
        g.close()
        print(json.dumps(out), flush=True)
        lines.append(out)
    with open(os.path.join(args.out, "bench_worklist_shapes.json"), "w") as f:
        json.dump(lines, f, indent=1)


def compare(a, b):
    ok = True
    for fn in sorted(f for f in os.listdir(a) if f.endswith(".npz")):
        x, y = np.load(os.path.join(a, fn)), np.load(os.path.join(b, fn))
        bad = []
        if not (x["counters"] == y["counters"]).all():
            bad.append("counters %s vs %s" % (x["counters"].tolist(), y["counters"].tolist()))
        if not (x["validity"] == y["validity"]).all():
            bad.append("validity")
        for j, fl in enumerate(x["is_float"]):
            u, v = x["values"][j], y["values"][j]
            if fl:
                uf, vf = u.view(np.float64), v.view(np.float64)
                if not (np.abs(uf - vf) <= 1e-12 * np.maximum(np.abs(vf), 1e-300)).all():
                    bad.append("output %d beyond 1e-12" % j)
            elif not (u == v).all():
                bad.append("output %d differs" % j)
        print("%s: %s" % (fn, "equal" if not bad else "; ".join(bad)))
        ok = ok and not bad
    return ok


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--shapes", default=",".join(SHAPES))
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--out", default=os.path.join(tempfile.gettempdir(), "bench_worklist_shapes"))
    ap.add_argument("--compare", nargs=2, metavar="DIR")
    args = ap.parse_args()
    if args.compare:
        sys.exit(0 if compare(*args.compare) else 1)
    measure(args)


if __name__ == "__main__":
    main()
