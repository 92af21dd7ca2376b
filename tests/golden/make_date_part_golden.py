#!/usr/bin/env python
"""Extract the reference's date_part / extract expectations into date_part_slt.json (data only: the inserted timestamps
and the expected rows of every `select date_part('<unit>', TIME)` and `select extract(<unit> from TIME)` query over the
five rows, with line citations).

Run next to a CnosDB v2.4.3 source tree (tests/test_calendar_parts.py only reads the JSON it writes):

    TSKV_REFERENCE=<path to the source tree> python tests/golden/make_date_part_golden.py
"""
import json
import os
import re

REF = os.environ["TSKV_REFERENCE"]
OUT = os.path.dirname(os.path.abspath(__file__))
DIR = "query_server/sqllogicaltests/cases/function/common/time_functions/"
QUERY = {"date_part.slt": r"select date_part\('(\w+)', TIME\) from test_date_part order by values asc;",
         "extract.slt": r"select extract\((\w+) from TIME\) from test_extract order by values asc;"}
UNITS = ["year", "quarter", "month", "week", "day", "hour", "minute", "second", "millisecond", "microsecond",
         "nanosecond", "dow", "doy", "epoch"]


def main():
    out = {"files": []}
    for name, pattern in QUERY.items():
        slt = DIR + name
        with open(os.path.join(REF, slt)) as f:
            txt = f.read()

        def line_of(pos):
            return txt.count("\n", 0, pos) + 1
        m = re.search(r"insert into test_\w+\(TIME, values\) values\n((?:\('[^']+', \d+\)[,;]\n)+)", txt)
        inserted = re.findall(r"\('([^']+)', (\d+)\)", m.group(1))
        assert len(inserted) == 5, inserted
        queries = []
        for q in re.finditer(r"query I\n" + pattern + r"\n----\n((?:[^\n]+\n){5})", txt):
            queries.append({"unit": q.group(1), "expected": q.group(2).split(),
                            "src": "%s:%d-%d" % (slt, line_of(q.start()), line_of(q.end()) - 1)})
        assert [x["unit"] for x in queries] == UNITS, queries
        out["files"].append({"src": "%s:%d-%d" % (slt, line_of(m.start()), line_of(m.end()) - 1),
                             "rows": [{"time": t, "values": int(v)} for t, v in inserted], "queries": queries})
        print(name, "queries:", len(queries))
    with open(os.path.join(OUT, "date_part_slt.json"), "w") as f:
        json.dump(out, f, indent=0)


if __name__ == "__main__":
    main()
