#!/usr/bin/env python
"""Extract the reference's increase(time, x ORDER BY time) expectations into increase_slt.json (data only, with line
citations): the two series of increase.slt's test_increase table and their `group by t0` answers, the rows of func_tb2
(read as make_stat_agg_golden.py reads them) with the answers for f0, f1 and f4, and the operand types the signature
refuses (f2 BOOLEAN, f3 STRING).

Run next to a CnosDB v2.4.3 source tree (tests/test_increase_reference.py and tests/test_gpu_increase.py only read the
JSON it writes):

    TSKV_REFERENCE=<path to the source tree> python tests/golden/make_increase_golden.py
"""
import json
import os
import re
import sys

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from make_stat_agg_golden import CASES, REF, line_of, tables  # noqa: E402

OUT = os.path.dirname(os.path.abspath(__file__))
SLT = CASES + "common/increase.slt"


def main():
    with open(os.path.join(REF, SLT)) as f:
        txt = f.read()
    series = []
    for m in re.finditer(r"INSERT INTO test_increase\.test_increase\(TIME, t0, f0\)\nVALUES\n((?:\s+\([^)]*\)[,;]\n)+)", txt):
        rows = [[v.strip().strip("'") for v in r.split(",")] for r in re.findall(r"\(([^)]*)\)", m.group(1))]
        series.append({"src": "%s:%d-%d" % (SLT, line_of(txt, m.start()), line_of(txt, m.end()) - 1),
                       "rows": [{"time": r[0], "t0": r[1], "f0": int(r[2])} for r in rows]})
    m = re.search(r"select t0, increase\(time, f0 order by time\) as increase\nfrom test_increase\.test_increase group by t0 "
                  r"order by t0, increase;\n----\n((?:\S+ \S+\n)+)", txt)
    grouped = {"src": "%s:%d" % (SLT, line_of(txt, m.start())),
               "expected": {a.strip('"'): int(b) for a, b in (ln.split() for ln in m.group(1).strip().split("\n"))}}
    answers = [{"column": q.group(1), "expected": q.group(2), "src": "%s:%d" % (SLT, line_of(txt, q.start()))}
               for q in re.finditer(r"select increase\(time, (f\d) order by time\) from func_tb2;\n----\n(\S+)", txt)]
    refused = [{"column": q.group(3), "type": q.group(1), "src": "%s:%d" % (SLT, line_of(txt, q.start(2)))}
               for q in re.finditer(r"argument types 'increase\\\(Timestamp\\\(Nanosecond, None\\\), (Boolean|Utf8)\\\)'[^\n]*\n"
                                    r"(select increase\(time, (f\d) order by time\) from func_tb2;)", txt)]
    out = {"test_increase": {"series": series, "group_by_t0": grouped}, "tables": {"func_tb2": tables()["func_tb2"]},
           "func_tb2": answers, "refused": refused}
    with open(os.path.join(OUT, "increase_slt.json"), "w") as f:
        json.dump(out, f, indent=1)
        f.write("\n")
    print("series:", len(series), "grouped:", grouped["expected"], "answers:", [(a["column"], a["expected"]) for a in answers],
          "refused:", [(r["column"], r["type"]) for r in refused])


if __name__ == "__main__":
    main()
