"""Writes tests/golden/compact_state_agg_slt.json from a CnosDB v2.4.3 source tree (data only, with line citations):

  - the `states` table of query_server/sqllogicaltests/cases/function/state_agg/state_agg.slt, its string states coded
    to i64 in order of first appearance (the scan takes integer states; the code keeps equality, which is all a map
    needs);
  - the answers of duration_in.slt that take no start time (compact_state_agg and state_agg alike), as nanoseconds;
  - the input_tuple_list / duration_tuple_list fixture of the unit tests in
    query_server/query/src/extension/expr/aggregate_function/state_agg/state_agg_data.rs ("111" -> 111 and so on);
  - the source line of each.

Run next to the source tree (tests/state_agg_reference.py and the golden tests only read the JSON):

    TSKV_REFERENCE=<path to the source tree> python tests/golden/make_compact_state_agg_golden.py
"""
import json
import os
import re
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
from make_stat_agg_golden import REF  # noqa: E402
SLT = "query_server/sqllogicaltests/cases/function/state_agg"
DATA_RS = "query_server/query/src/extension/expr/aggregate_function/state_agg/state_agg_data.rs"


def interval_ns(s):
    y, mo, d, h, mi, sec = re.fullmatch(r"(-?\d+) years (-?\d+) mons (-?\d+) days (-?\d+) hours (-?\d+) mins (-?[\d.]+) secs", s).groups()
    assert int(y) == 0 and int(mo) == 0, s
    whole, _, frac = sec.partition(".")
    return ((int(d) * 24 + int(h)) * 60 + int(mi)) * 60_000_000_000 + int(whole) * 1_000_000_000 + int((frac + "000000000")[:9])


def ts_ns(s):
    return int(np.datetime64(s.replace(" ", "T"), "ns").astype(np.int64))


def states_table(root):
    path = os.path.join(root, SLT, "state_agg.slt")
    rows, codes = [], {}
    for no, line in enumerate(open(path), 1):
        m = re.match(r"\s*\('([^']+)', '([^']+)'\)[,;]", line)
        if m:
            code = codes.setdefault(m.group(2), len(codes))
            rows.append({"line": no, "time": ts_ns(m.group(1)), "state": m.group(2), "code": code})
    return {"src": "%s/state_agg.slt" % SLT, "rows": rows, "codes": codes}


def duration_answers(root, codes):
    path = os.path.join(root, SLT, "duration_in.slt")
    lines = open(path).read().splitlines()
    out = []
    for i, line in enumerate(lines):
        m = re.match(r"select duration_in\((compact_state_agg|state_agg)\(time, state\), '(\w+)'\) from states;", line)
        if m:
            assert lines[i + 1] == "----", lines[i + 1]
            out.append({"src": "%s/duration_in.slt:%d" % (SLT, i + 1), "sql": line, "agg": m.group(1), "state": m.group(2),
                        "code": codes[m.group(2)], "expected": interval_ns(lines[i + 2]), "expected_text": lines[i + 2]})
    return out


def unit_fixture(root):
    src = open(os.path.join(root, DATA_RS)).read()

    def block(name):
        a = src.index("fn %s()" % name)
        body = src[a:src.index("\n    }\n", a)]
        return a, body

    a, inp = block("input_tuple_list")
    pts = re.findall(r"TimestampNanosecond\(Some\((\d+)\), None\),\s*ScalarValue::Utf8\(Some\(\"(\d+)\"", inp)
    b, dur = block("duration_tuple_list")
    durs = re.findall(r"Utf8\(Some\(\"(\d+)\"\.to_string\(\)\)\),\s*ScalarValue::IntervalMonthDayNano\(Some\((\d+)\)\)", dur)
    return {"src": "%s:%d-%d" % (DATA_RS, src[:a].count("\n") + 1, src[:b].count("\n") + 1),
            "points": [[int(t), int(s)] for t, s in pts], "durations": [[int(s), int(d)] for s, d in durs]}


def main():
    root = REF
    tbl = states_table(root)
    g = {"states": tbl, "answers": duration_answers(root, tbl["codes"]), "unit": unit_fixture(root)}
    assert len(g["answers"]) == 2 and len(g["unit"]["points"]) == 6 and len(g["unit"]["durations"]) == 3, g
    with open(os.path.join(HERE, "compact_state_agg_slt.json"), "w") as f:
        json.dump(g, f, indent=1)
        f.write("\n")


if __name__ == "__main__":
    main()
