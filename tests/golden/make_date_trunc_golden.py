#!/usr/bin/env python
"""Extract the reference's date_trunc expectations into date_trunc_slt.json (data only: the inserted timestamps and the
expected rows of the eight `select date_trunc('<unit>', TIME)` queries, with line citations).

Run next to a CnosDB v2.4.3 source tree (tests/test_calendar_edges.py only reads the JSON it writes):

    TSKV_REFERENCE=<path to the source tree> python tests/golden/make_date_trunc_golden.py
"""
import json
import os
import re

REF = os.environ["TSKV_REFERENCE"]
OUT = os.path.dirname(os.path.abspath(__file__))
SLT = "query_server/sqllogicaltests/cases/function/common/time_functions/date_trunc.slt"
UNITS = ["year", "quarter", "month", "week", "day", "hour", "minute", "second"]


def main():
    with open(os.path.join(REF, SLT)) as f:
        txt = f.read()

    def line_of(pos):
        return txt.count("\n", 0, pos) + 1
    m = re.search(r"insert into test_date_trunc\(TIME, values\) values\n((?:\('[^']+', \d+\)[,;]\n)+)", txt)
    inserted = re.findall(r"\('([^']+)', (\d+)\)", m.group(1))
    assert len(inserted) == 5, inserted
    queries = []
    for q in re.finditer(r"query I\nselect date_trunc\('(\w+)', TIME\) from test_date_trunc order by values asc;\n----\n"
                         r"((?:[^\n]+\n){5})", txt):
        queries.append({"unit": q.group(1), "expected": q.group(2).split(),
                        "src": "%s:%d-%d" % (SLT, line_of(q.start()), line_of(q.end()) - 1)})
    assert [x["unit"] for x in queries] == UNITS, queries
    with open(os.path.join(OUT, "date_trunc_slt.json"), "w") as f:
        json.dump({"src": "%s:%d-%d" % (SLT, line_of(m.start()), line_of(m.end()) - 1),
                   "rows": [{"time": t, "values": int(v)} for t, v in inserted], "queries": queries}, f, indent=0)
    print("date_trunc queries:", len(queries))


if __name__ == "__main__":
    main()
