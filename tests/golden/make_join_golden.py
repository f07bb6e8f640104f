"""Regenerates tests/golden/join_tables.json: the two tables of the reference's join tests (src/dataframe.rs:1005-1060 read them
from a Postgres server), taken from the SQL script that creates them.

Run with a checkout of the reference (the tests themselves only read the JSON this writes):
    python tests/golden/make_join_golden.py <reference checkout>/sql/postgresql/002.sql
Every `insert into <table> (<columns>) values (...), ...;` of the script becomes a table of columns.  Float columns are written
as float.hex() strings ('inf', 'nan') so that the file stays strict JSON; a quoted 'infinity' / 'NaN' is Postgres's float literal.
"""
import json
import os
import re
import sys

HERE = os.path.dirname(os.path.abspath(__file__))


def _sql_value(tok):
    tok = tok.strip()
    if tok.lower() == "null":
        return None
    if tok.startswith("'"):
        return tok[1:-1]
    return int(tok) if re.fullmatch(r"-?\d+", tok) else float(tok)


def main():
    with open(sys.argv[1]) as f:
        sql = f.read()
    out = {"source": "reference sql/postgresql/002.sql (the data of the join tests, src/dataframe.rs:1005-1060)"}
    for table, cols, body in re.findall(r"insert into (\w+) \(([^)]*)\)\s*values\s*(.*?);", sql, re.S | re.I):
        names = [c.strip() for c in cols.split(",")]
        rows = [[_sql_value(t) for t in re.findall(r"'[^']*'|[^,]+", row)] for row in re.findall(r"\(([^)]*)\)", body)]
        table_out = {}
        for j, name in enumerate(names):
            col = [r[j] for r in rows]
            if any(isinstance(v, float) for v in col) or name == "f":   # double precision: 'infinity' / 'NaN' arrive as text
                col = [None if v is None else float(v).hex() for v in col]
            table_out[name] = col
        out[table] = table_out
    with open(os.path.join(HERE, "join_tables.json"), "w") as f:
        json.dump(out, f, indent=1)
    print("wrote join_tables.json:", ", ".join(f"{t} {len(next(iter(out[t].values())))} rows" for t in out if t != "source"))


if __name__ == "__main__":
    main()
