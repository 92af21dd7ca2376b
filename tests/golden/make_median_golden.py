#!/usr/bin/env python
"""Extract the reference's exact-median expectations into median_slt.json (data only, with line citations): the table
test_approx_median_tbl of approx_median.slt (its CREATE TABLE types and the rows of its first INSERT) and every
`SELECT median(col)` query that runs before the next INSERT, with its expected value. (The file's approx_median checks
are t-digest estimates, and its later checks run after more rows arrive: neither is extracted.)

Run next to a CnosDB v2.4.3 source tree (tests/test_median_reference.py and tests/test_gpu_median.py only read the JSON
it writes):

    TSKV_REFERENCE=<path to the source tree> python tests/golden/make_median_golden.py
"""
import json
import os
import re
import sys

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from make_stat_agg_golden import CASES, REF, line_of  # noqa: E402

OUT = os.path.dirname(os.path.abspath(__file__))
SLT = CASES + "common/approx_agg/approx_median.slt"


def main():
    with open(os.path.join(REF, SLT)) as f:
        txt = f.read()
    c = re.search(r"CREATE TABLE test_approx_median_tbl \(\n((?:\s+\w+ [\w ]+,?\n)+)\);", txt)
    types = {m.group(1): m.group(2).strip() for m in re.finditer(r"(\w+) ([\w ]+?),?\n", c.group(1))}
    m = re.search(r"INSERT INTO test_approx_median_tbl\(time, val, s_val, d_val, b_val, u_val\) VALUES\n((?:\([^)]*\)[,;]\n)+)", txt)
    rows = [[v.strip().strip("'") for v in r.split(",")] for r in re.findall(r"\(([^)]*)\)", m.group(1))]
    table = {"src": "%s:%d-%d" % (SLT, line_of(txt, m.start()), line_of(txt, m.end()) - 1),
             "types_src": "%s:%d-%d" % (SLT, line_of(txt, c.start()), line_of(txt, c.end())),
             "columns": ["time", "val", "s_val", "d_val", "b_val", "u_val"], "types": types, "rows": rows}
    next_insert = txt.index("INSERT", m.end())
    checks = []
    for q in re.finditer(r"query \w*\s*\nSELECT median\((\w+)\)\s+FROM test_approx_median_tbl;\n----\n(\S+)", txt):
        if q.start() > next_insert:
            continue
        checks.append({"column": q.group(1), "expected": q.group(2),
                       "src": "%s:%d-%d" % (SLT, line_of(txt, q.start()), line_of(txt, q.end()))})
    print("rows:", len(rows), "checks:", len(checks))
    with open(os.path.join(OUT, "median_slt.json"), "w") as f:
        json.dump({"table": table, "checks": checks}, f, indent=1)


if __name__ == "__main__":
    main()
