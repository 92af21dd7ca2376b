#!/usr/bin/env python
"""Extract the reference's covariance / correlation expectations into covar_slt.json (data only, with line citations):
the rows of func_tb2 (read as make_stat_agg_golden.py reads them), every `abs(F(a, b) -/+ value) < tolerance` check of
corr.slt, covar.slt, covar_pop.slt and covar_samp.slt (operands may be `-f1`), the `F(1, 2)` constants, the queries that
return NULL, the refused input types, and the rows and expected values of the `unorder` table of unorderdata_func.slt.

Run next to a CnosDB v2.4.3 source tree (tests/test_covar_reference.py and tests/test_gpu_covariance.py only read the
JSON it writes):

    TSKV_REFERENCE=<path to the source tree> python tests/golden/make_covar_golden.py
"""
import json
import os
import re
import sys

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from make_stat_agg_golden import CASES, REF, line_of, tables  # noqa: E402

OUT = os.path.dirname(os.path.abspath(__file__))
FILES = ["corr", "covar", "covar_pop", "covar_samp"]


def unorder():
    src = CASES + "common/unorderdata_func.slt"
    with open(os.path.join(REF, src)) as f:
        txt = f.read()
    m = re.search(r"INSERT INTO unorder \(TIME, x, y\) VALUES\n((?:\s+\([^)]*\)[,;]\n)+)", txt)
    rows = [[v.strip().strip("'") for v in r.split(",")] for r in re.findall(r"\(([^)]*)\)", m.group(1))]
    out = {"src": "%s:%d-%d" % (src, line_of(txt, m.start()), line_of(txt, m.end()) - 1), "columns": ["time", "x", "y"],
           "types": {"x": "DOUBLE", "y": "DOUBLE"}, "rows": rows, "expected": []}
    for q in re.finditer(r"SELECT (corr|covar|covar_pop|covar_samp)\(x, y\) FROM unorder;\n----\n(\S+)", txt):
        out["expected"].append({"func": q.group(1), "value": float(q.group(2)), "src": "%s:%d" % (src, line_of(txt, q.start()))})
    return out


def main():
    out = {"tables": {"func_tb2": tables()["func_tb2"]}, "checks": [], "constants": [], "nulls": [], "refused": [],
           "unorder": unorder()}
    for name in FILES:
        slt = CASES + "common/statistical_agg/%s.slt" % name
        with open(os.path.join(REF, slt)) as f:
            txt = f.read()
        for q in re.finditer(r"select abs\((\w+)\((-?\w+), (-?\w+)\) ([-+]) ([0-9.e]+) ?\) < ([0-9.e]+) +from (\w+);\n----\ntrue", txt):
            v = float(q.group(5))  # abs(F - v) < tol, written as `F - v` or `F + (-v)`
            out["checks"].append({"func": q.group(1), "x": q.group(2), "y": q.group(3), "value": v if q.group(4) == "-" else -v,
                                  "tolerance": float(q.group(6)), "table": q.group(7),
                                  "src": "%s:%d" % (slt, line_of(txt, q.start()))})
        for q in re.finditer(r"select (\w+)\(1, 2\) from (\w+);\n----\n(\S+)", txt):
            out["constants"].append({"func": q.group(1), "table": q.group(2), "expected": q.group(3),
                                     "src": "%s:%d" % (slt, line_of(txt, q.start()))})
        for q in re.finditer(r"select (\w+)\((\w+), (\w+)\) from (\w+);\n----\nNULL", txt):
            out["nulls"].append({"func": q.group(1), "x": q.group(2), "y": q.group(3), "table": q.group(4),
                                 "src": "%s:%d" % (slt, line_of(txt, q.start()))})
        for q in re.finditer(r"does not support inputs of type (Timestamp|Utf8)\\?[^\n]*\n(select (\w+)\((\w+), (\w+)\) from (\w+);)", txt):
            out["refused"].append({"func": q.group(3), "x": q.group(4), "y": q.group(5), "table": q.group(6), "type": q.group(1),
                                   "src": "%s:%d" % (slt, line_of(txt, q.start(2)))})
    print("checks:", len(out["checks"]), "constants:", len(out["constants"]), "nulls:", len(out["nulls"]),
          "refused:", len(out["refused"]), "unorder rows:", len(out["unorder"]["rows"]),
          "unorder values:", len(out["unorder"]["expected"]))
    with open(os.path.join(OUT, "covar_slt.json"), "w") as f:
        json.dump(out, f, indent=0)


if __name__ == "__main__":
    main()
