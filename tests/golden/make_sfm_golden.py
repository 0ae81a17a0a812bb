"""Generates tests/golden/sfm_schema.json: the PRAGMA table_info, foreign_key_list and index_list rows (and each
index's index_info) of an empty database made by the REFERENCE's create_empty_db (the reference's
sfm/import_feature_matches.py with sfm/colmap_utils/database.py).  Needs a ParticleSfM checkout at $PSFM_REFERENCE:
    python tests/golden/make_sfm_golden.py
"""
import json
import os
import sys
import tempfile
import types

HERE = os.path.dirname(os.path.abspath(__file__))


def schema_rows(con):
    """{table: {"columns", "foreign_keys", "indexes"}} of an open sqlite3 connection, every row as a list."""
    out = {}
    tables = [r[0] for r in con.execute("SELECT name FROM sqlite_master WHERE type = 'table' AND name NOT LIKE 'sqlite_%' "
                                        "ORDER BY name")]
    for t in tables:
        idx = [list(r) for r in con.execute(f"PRAGMA index_list({t})")]
        out[t] = {"columns": [list(r) for r in con.execute(f"PRAGMA table_info({t})")],
                  "foreign_keys": [list(r) for r in con.execute(f"PRAGMA foreign_key_list({t})")],
                  "indexes": sorted(idx, key=lambda r: r[1]),
                  "index_columns": {r[1]: [list(c) for c in con.execute(f"PRAGMA index_info({r[1]})")] for r in idx}}
    return out


def main():
    import sqlite3
    sys.path.insert(0, os.path.join(os.environ["PSFM_REFERENCE"], "sfm"))
    # the reference module's other imports (the trajectory reader) are not needed to create the schema
    sys.modules.setdefault("matches_from_flow", types.SimpleNamespace(traj_to_matches=None))
    import import_feature_matches as ref
    with tempfile.TemporaryDirectory() as td:
        path = os.path.join(td, "database.db")
        ref.create_empty_db(path)
        con = sqlite3.connect(path)
        rows = schema_rows(con)
        con.close()
    with open(os.path.join(HERE, "sfm_schema.json"), "w") as f:
        json.dump(rows, f, indent=1, sort_keys=True)
        f.write("\n")
    print(sorted(rows))


if __name__ == "__main__":
    main()
