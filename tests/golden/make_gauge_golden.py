#!/usr/bin/env python
"""Extract the reference's gauge_agg expectations into gauge_slt.json (data only, with line citations):
- the tables: setup.slt's func_tbl and func_tb2, rate.slt's func_rate_tbl (its three INSERTs, in order: each answer
  names how many of its rows were inserted before it), the idelta tables of idelta_left.slt / idelta_right.slt and
  gauge_agg.slt's `unorder` table;
- every answered query of function/gauge/*.slt whose select list holds gauge_agg(time, x) or an accessor of it
  (delta, rate, time_delta, idelta_left, idelta_right, first_time, first_val, last_time, last_val), with its SQL and the
  answer's lines as printed;
- the operand types gauge_agg refuses at planning (Boolean, Utf8, Timestamp).

Run next to a CnosDB v2.4.3 source tree (tests/gauge_reference.py and the gauge golden tests only read the JSON):

    TSKV_REFERENCE=<path to the source tree> python tests/golden/make_gauge_golden.py
"""
import json
import os
import re
import sys

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from make_stat_agg_golden import CASES, REF, line_of, tables  # noqa: E402

OUT = os.path.dirname(os.path.abspath(__file__))
GAUGE = CASES + "gauge/"
FILES = ("gauge_agg", "delta", "rate", "time_delta", "idelta_left", "idelta_right", "first_time", "first_val", "last_time",
         "last_val")


def read(path):
    with open(os.path.join(REF, path)) as f:
        return f.read()


def rows_of(block):
    return [[v.strip().strip("'") for v in r.split(",")] for r in re.findall(r"\(([^)]*)\)", block)]


def inserts(txt, path, table):
    """[(src, columns, rows)] of every INSERT into `table` in txt, in order."""
    out = []
    pat = r"INSERT (?:INTO )?%s ?\(([^)]*)\)\s*\nVALUES\n((?:\s*\([^)]*\)[,;]?\n)+)" % table
    for m in re.finditer(pat, txt):
        cols = [c.strip().lower() for c in m.group(1).split(",")]
        out.append({"src": "%s:%d-%d" % (path, line_of(txt, m.start()), line_of(txt, m.end()) - 1), "columns": cols,
                    "rows": rows_of(m.group(2))})
    return out


def main():
    base = tables()
    out_tables = {"func_tbl": base["func_tbl"], "func_tb2": base["func_tb2"]}
    answers, refused = [], []
    for name in FILES:
        path = GAUGE + name + ".slt"
        txt = read(path)
        for m in re.finditer(r"CREATE TABLE(?: IF NOT EXISTS)? (\w+)\s*\(([^;]*)\);", txt):
            table = m.group(1)
            ins = inserts(txt, path, table)
            if not ins:
                continue
            types = {}
            for part in re.split(r",(?![^(]*\))", m.group(2)):
                part = part.strip()
                if part.upper().startswith("TAGS"):
                    continue
                col, typ = part.split(None, 1)
                types[col.lower()] = typ.strip().upper()
            out_tables[table] = {"src": "%s:%d" % (path, line_of(txt, m.start())), "columns": ins[0]["columns"],
                                 "types": types, "rows": [r for i in ins for r in i["rows"]],
                                 "inserts": [{"src": i["src"], "n_rows": len(i["rows"])} for i in ins]}
        for m in re.finditer(r"\nquery[^\n]*\n(select[^\n]*)\n----\n((?:[^\n]+\n)+)", txt, flags=re.I):
            sql = m.group(1).strip()
            if "gauge_agg(" not in sql.lower():
                continue
            table = re.search(r"from (\w+)", sql, flags=re.I).group(1)
            entry = {"src": "%s:%d" % (path, line_of(txt, m.start() + 1)), "sql": sql, "table": table,
                     "expected": m.group(2).rstrip("\n").split("\n")}
            if table in out_tables and "inserts" in out_tables[table]:  # rows inserted before this query
                before = [i for i in inserts(txt[:m.start()], path, table)]
                entry["n_rows"] = sum(len(i["rows"]) for i in before)
            answers.append(entry)
        for m in re.finditer(r"(?:statement|query) error [^\n]*argument types 'gauge_agg\\\(Timestamp\\\(Nanosecond, None\\\), "
                             r"(\w+)[^\n]*\n(select[^\n]*)", txt):
            refused.append({"src": "%s:%d" % (path, line_of(txt, m.start())), "type": m.group(1), "sql": m.group(2).strip()})
    out = {"tables": out_tables, "answers": answers, "refused": refused}
    with open(os.path.join(OUT, "gauge_slt.json"), "w") as f:
        json.dump(out, f, indent=1)
        f.write("\n")
    print("tables:", {k: len(v["rows"]) for k, v in out_tables.items()}, "answers:", len(answers),
          "refused:", sorted({r["type"] for r in refused}))


if __name__ == "__main__":
    main()
