#!/usr/bin/env python
"""Extract the reference's variance / standard deviation expectations into stat_agg_slt.json (data only: the rows of
func_tbl and func_tb2 the six statistical_agg files read, every `abs(F(col) - value) < tolerance` check, the constant
argument cases and the refused input types, with line citations).

Run next to a CnosDB v2.4.3 source tree (tests/test_stat_agg_reference.py only reads the JSON it writes):

    TSKV_REFERENCE=<path to the source tree> python tests/golden/make_stat_agg_golden.py
"""
import json
import os
import re

REF = os.environ["TSKV_REFERENCE"]
OUT = os.path.dirname(os.path.abspath(__file__))
CASES = "query_server/sqllogicaltests/cases/function/"
FILES = ["stddev", "stddev_pop", "stddev_samp", "var", "var_pop", "var_samp"]


def line_of(txt, pos):
    return txt.count("\n", 0, pos) + 1


def tables():
    src = CASES + "setup.slt"
    with open(os.path.join(REF, src)) as f:
        txt = f.read()
    out = {}
    for name, pattern in (("func_tbl", r"INSERT func_tbl\(TIME, f0, f1, t0, t1\)\nVALUES\n((?:\s+\([^)]*\)[,;]\n)+)"),
                          ("func_tb2", r"INSERT INTO func_tb2\(TIME, f0, f1, f2, f3, f4, t0, t1, t2\) \nVALUES\n((?:\s+\([^)]*\)[,;]\n)+)")):
        m = re.search(pattern, txt)
        rows = [[v.strip().strip("'") for v in r.split(",")] for r in re.findall(r"\(([^)]*)\)", m.group(1))]
        out[name] = {"src": "%s:%d-%d" % (src, line_of(txt, m.start()), line_of(txt, m.end()) - 1), "rows": rows}
    out["func_tbl"]["columns"] = ["time", "f0", "f1", "t0", "t1"]
    out["func_tbl"]["types"] = {"f0": "BIGINT", "f1": "BIGINT"}
    out["func_tb2"]["columns"] = ["time", "f0", "f1", "f2", "f3", "f4", "t0", "t1", "t2"]
    out["func_tb2"]["types"] = {"f0": "BIGINT UNSIGNED", "f1": "DOUBLE", "f2": "BOOLEAN", "f3": "STRING", "f4": "BIGINT"}
    return out


def main():
    out = {"tables": tables(), "checks": [], "constants": [], "refused": []}
    for name in FILES:
        slt = CASES + "common/statistical_agg/%s.slt" % name
        with open(os.path.join(REF, slt)) as f:
            txt = f.read()
        for q in re.finditer(r"select abs\((\w+)\((\w+)\) - ([-0-9.e]+)\) < ([0-9.e]+) +from (\w+);\n----\ntrue", txt):
            out["checks"].append({"func": q.group(1), "column": q.group(2), "value": float(q.group(3)),
                                  "tolerance": float(q.group(4)), "table": q.group(5),
                                  "src": "%s:%d" % (slt, line_of(txt, q.start()))})
        for q in re.finditer(r"select (\w+)\(1\) from (\w+);\n----\n(\S+)", txt):
            out["constants"].append({"func": q.group(1), "table": q.group(2), "expected": q.group(3),
                                     "src": "%s:%d" % (slt, line_of(txt, q.start()))})
        for q in re.finditer(r"does not support inputs of type (Boolean|Utf8)\\\..*\n(select (\w+)\((\w+)\) from (\w+);)", txt):
            out["refused"].append({"func": q.group(3), "column": q.group(4), "table": q.group(5), "type": q.group(1),
                                   "src": "%s:%d" % (slt, line_of(txt, q.start(2)))})
    print("checks:", len(out["checks"]), "constants:", len(out["constants"]), "refused:", len(out["refused"]))
    with open(os.path.join(OUT, "stat_agg_slt.json"), "w") as f:
        json.dump(out, f, indent=0)


if __name__ == "__main__":
    main()
