#!/usr/bin/env python
"""Extract the reference's mode(x) and distinct-count expectations into mode_slt.json (data only, with line citations):
- mode.slt over func_tbl (setup.slt's rows and mode.slt's INSERT): mode(f1), mode(f0) and mode(f0) group by t0;
- mode.slt over func_tb3 (setup.slt's rows, their time and scalar columns): the bigint, unsigned and double answers,
  and the operand types the scan refuses (TIME, BOOLEAN, STRING, geometry);
- approx_distinct.slt over tbl_with_nulls: approx_distinct(val) and approx_distinct(u_val). On these few values the
  HyperLogLog estimate equals the exact distinct count.

Run next to a CnosDB v2.4.3 source tree (tests/test_mode_reference.py and tests/test_gpu_mode_golden.py only read the
JSON it writes):

    TSKV_REFERENCE=<path to the source tree> python tests/golden/make_mode_golden.py
"""
import json
import os
import re
import sys

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from make_stat_agg_golden import CASES, REF, line_of, tables  # noqa: E402

OUT = os.path.dirname(os.path.abspath(__file__))
MODE = CASES + "common/mode.slt"
SETUP = CASES + "setup.slt"
DISTINCT = CASES + "common/approx_agg/approx_distinct.slt"


def read(path):
    with open(os.path.join(REF, path)) as f:
        return f.read()


def rows_of(block):
    return [[v.strip().strip("'") for v in r.split(",")] for r in re.findall(r"\(([^)]*)\)", block)]


def func_tb3():
    """The time, tag and scalar field columns of setup.slt's func_tb3 rows (the geometry literals that follow are left
    out)."""
    txt = read(SETUP)
    rows = []
    pat = (r"\('(\d{4}-[^']+)', '(\w+)', '(\w+)', '(\w+)', '(\w+)', ([-\w.]+), ([-\w.]+), (\w+), '([^']*)', ([-\w.]+), ")
    for m in re.finditer(pat, txt):
        rows.append({"line": line_of(txt, m.start()), "time": m.group(1), "t0": m.group(2), "f0_bigint": int(m.group(6)),
                     "f1_bigint_unsign": int(m.group(7)), "f2_boolean": m.group(8), "f3_string": m.group(9),
                     "f4_double": float(m.group(10))})
    return {"src": "%s:%d-%d" % (SETUP, rows[0]["line"], rows[-1]["line"]), "rows": rows}


def main():
    txt = read(MODE)
    m = re.search(r"INSERT func_tbl\(TIME, f0, f1, t0, t1\)\nVALUES\n((?:\s+\([^)]*\)[,;]\n)+)", txt)
    extra = {"src": "%s:%d-%d" % (MODE, line_of(txt, m.start()), line_of(txt, m.end()) - 1), "rows": rows_of(m.group(1))}
    ungrouped = [{"column": q.group(1), "expected": int(q.group(2)), "src": "%s:%d" % (MODE, line_of(txt, q.start()))}
                 for q in re.finditer(r"select mode\((f\d)\) from func_tbl;\n----\n(\d+)", txt)]
    q = re.search(r"select mode\((f\d)\) from func_tbl group by t0 order by t0;\n----\n((?:\d+\n)+)", txt)
    by_t0 = {"column": q.group(1), "expected": [int(v) for v in q.group(2).split()], "src": "%s:%d" % (MODE, line_of(txt, q.start()))}
    tb3 = []
    for q in re.finditer(r"select mode\((\w+)\) from func_tb3 where \w+ in \(([^)]*)\);\n----\n(\S+)", txt):
        tb3.append({"column": q.group(1), "in": q.group(2).strip("'"), "expected": q.group(3).strip('"'),
                    "src": "%s:%d" % (MODE, line_of(txt, q.start()))})
    for q in re.finditer(r"select mode\((loc\w+)\) from func_tb3 where \w+ in \('([^']*)'\);\n----\n(.+)", txt):
        tb3.append({"column": q.group(1), "in": q.group(2), "expected": q.group(3).strip('"'),
                    "src": "%s:%d" % (MODE, line_of(txt, q.start()))})
    pushed = {"f0_bigint": "BIGINT", "f1_bigint_unsign": "BIGINT UNSIGNED", "f4_double": "DOUBLE"}
    answers = [a for a in tb3 if a["column"] in pushed]
    refused = [dict(a, type={"time": "TIME", "f2_boolean": "BOOLEAN", "f3_string": "STRING"}.get(a["column"], "GEOMETRY"))
               for a in tb3 if a["column"] not in pushed]
    dtxt = read(DISTINCT)
    m = re.search(r"INSERT INTO tbl_with_nulls \(time, val, s_val, d_val, b_val, u_val\) VALUES\n((?:\([^)]*\)[,;]\n)+)", dtxt)
    nulls = {"src": "%s:%d-%d" % (DISTINCT, line_of(dtxt, m.start()), line_of(dtxt, m.end()) - 1),
             "columns": ["time", "val", "s_val", "d_val", "b_val", "u_val"], "types": {"val": "BIGINT", "u_val": "BIGINT UNSIGNED"},
             "rows": rows_of(m.group(1))}
    distinct = [{"column": q.group(1), "expected": int(q.group(2)), "src": "%s:%d" % (DISTINCT, line_of(dtxt, q.start()))}
                for q in re.finditer(r"SELECT approx_distinct\((val|u_val)\) FROM tbl_with_nulls;\n----\n(\d+)", dtxt)]
    base = tables()["func_tbl"]
    out = {"func_tbl": {"setup": base, "mode_insert": extra, "columns": base["columns"], "types": base["types"]},
           "func_tbl_modes": ungrouped, "func_tbl_mode_by_t0": by_t0,
           "func_tb3": dict(func_tb3(), types=pushed), "func_tb3_modes": answers, "refused": refused,
           "tbl_with_nulls": nulls, "distinct": distinct}
    with open(os.path.join(OUT, "mode_slt.json"), "w") as f:
        json.dump(out, f, indent=1)
        f.write("\n")
    print("func_tbl rows:", len(base["rows"]) + len(extra["rows"]), "modes:", [(a["column"], a["expected"]) for a in ungrouped],
          "by t0:", by_t0["expected"], "func_tb3 rows:", len(out["func_tb3"]["rows"]),
          "answers:", [(a["column"], a["expected"]) for a in answers], "refused:", [(r["column"], r["type"]) for r in refused],
          "distinct:", [(a["column"], a["expected"]) for a in distinct])


if __name__ == "__main__":
    main()
