"""Writes tests/golden/state_agg_periods_slt.json from a CnosDB v2.4.3 source tree (data only, with line citations):

  - the `states` table of query_server/sqllogicaltests/cases/function/state_agg/state_agg.slt, coded to i64 as
    make_compact_state_agg_golden.py codes it (in order of first appearance);
  - the answers of state_at.slt (the state's code, or null for the "NULL" answer) and its compact_state_agg error;
  - the answers of duration_in.slt that take a start time, with and without an interval (as nanoseconds), and its
    compact_state_agg errors;
  - the input_tuple_list / period_tuple_list fixture of the unit tests in
    query_server/query/src/extension/expr/aggregate_function/state_agg/state_agg_data.rs ("111" -> 111 and so on);
  - the source line of each.

Run next to the source tree (tests/state_periods_reference.py and the golden tests only read the JSON):

    TSKV_REFERENCE=<path to the source tree> python tests/golden/make_state_agg_golden.py
"""
import json
import os
import re
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
from make_compact_state_agg_golden import DATA_RS, SLT, interval_ns, states_table, ts_ns  # noqa: E402
from make_stat_agg_golden import REF  # noqa: E402


def _queries(root, name):
    """(line number, sql, the lines after it) of every query of an slt file, its sql joined over its lines."""
    lines = open(os.path.join(root, SLT, name)).read().splitlines()
    out = []
    i = 0
    while i < len(lines):
        if lines[i].startswith("query "):
            head, j = lines[i], i + 1
            sql = []
            while j < len(lines) and lines[j] and lines[j] != "----":
                sql.append(lines[j].strip())
                j += 1
            out.append((i + 2, head, " ".join(sql), lines[j + 1] if j < len(lines) and lines[j] == "----" else None))
            i = j
        i += 1
    return out


def state_at_answers(root, codes):
    out = []
    for no, head, sql, ans in _queries(root, "state_at.slt"):
        m = re.fullmatch(r"select state_at\((compact_state_agg|state_agg)\(time, state\), Timestamp '([^']+)'\) from states;", sql)
        assert m, sql
        e = {"src": "%s/state_at.slt:%d" % (SLT, no), "sql": sql, "agg": m.group(1), "ts": ts_ns(m.group(2))}
        if head.startswith("query error"):
            e["error"] = re.search(r"err: (.*?doesn't support compact_agg)", head).group(1).replace("\\", "")
        else:
            state = ans.strip('"')
            e["expected_text"] = ans
            e["expected"] = None if state == "NULL" else codes[state]
        out.append(e)
    return out


def duration_answers(root, codes):
    out = []
    for no, head, sql, ans in _queries(root, "duration_in.slt"):
        m = re.fullmatch(r"select duration_in\((compact_state_agg|state_agg)\(time, state\), '(\w+)', Timestamp '([^']+)'"
                         r"(?:, interval '(\d+) day')?\) from states;", sql)
        if not m:
            continue
        e = {"src": "%s/duration_in.slt:%d" % (SLT, no), "sql": sql, "agg": m.group(1), "state": m.group(2),
             "code": codes[m.group(2)], "start": ts_ns(m.group(3)),
             "interval": None if m.group(4) is None else int(m.group(4)) * 86_400_000_000_000}
        if head.startswith("query error"):
            e["error"] = re.search(r"err: (.*?doesn't support compact_agg)", head).group(1).replace("\\", "")
        else:
            e["expected"] = interval_ns(ans)
            e["expected_text"] = ans
        out.append(e)
    return out


def unit_fixture(root):
    src = open(os.path.join(root, DATA_RS)).read()

    def block(name):
        a = src.index("fn %s()" % name)
        return a, src[a:src.index("\n    }\n", a)]

    a, inp = block("input_tuple_list")
    pts = re.findall(r"TimestampNanosecond\(Some\((\d+)\), None\),\s*ScalarValue::Utf8\(Some\(\"(\d+)\"", inp)
    b, per = block("period_tuple_list")
    periods = []
    for state, body in re.findall(r"Utf8\(Some\(\"(\d+)\"\.to_string\(\)\)\),\s*vec!\[(.*?)\],\s*\)", per, re.S):
        ts = [int(t) for t in re.findall(r"TimestampNanosecond\(Some\((\d+)\), None\)", body)]
        periods.append([int(state), [[ts[i], ts[i + 1]] for i in range(0, len(ts), 2)]])
    return {"src": "%s:%d-%d" % (DATA_RS, src[:a].count("\n") + 1, src[:b].count("\n") + 1),
            "points": [[int(t), int(s)] for t, s in pts], "periods": periods}


def main():
    root = REF
    tbl = states_table(root)
    g = {"states": tbl, "state_at": state_at_answers(root, tbl["codes"]),
         "duration_in": duration_answers(root, tbl["codes"]), "unit": unit_fixture(root)}
    assert len(g["state_at"]) == 5 and len(g["duration_in"]) == 4, g
    assert len(g["unit"]["points"]) == 6 and [len(p) for _, p in g["unit"]["periods"]] == [2, 2, 1], g["unit"]
    with open(os.path.join(HERE, "state_agg_periods_slt.json"), "w") as f:
        json.dump(g, f, indent=1)
        f.write("\n")


if __name__ == "__main__":
    main()
