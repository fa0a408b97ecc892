#!/usr/bin/env python
"""Build the lookup tables used by both the oracle and the CUDA library into mortal_b200/data/ (git-ignored build
products, like the built .so).

* shanten_suhai.bin / shanten_jihai.bin are GENERATED from first principles by tools/gen_shanten_tables.cc (a DP over
  the rank counts; no input files) and truncated to the row counts of libriichi's tables (1,940,777 / 78,032 rows:
  indices past the end read as an all-zero row in the reference, algo/shanten.rs:52, and that quirk is part of the
  contract). The result is checked byte for byte against libriichi's data files (tests/golden/tables/).
* agari.bin (9,362 keys) is GENERATED from first principles by tools/gen_agari_table.py (enumeration of all hand shapes
  that split into melds + pair or seven pairs; no input files). Records are written in ascending key order; the result
  is checked against libriichi's data file (tests/golden/tables/) as key -> ordered div list (the
  reference loads its file into a hash map, agari.rs:22-51, so the order of records is not content).
Nothing is copied from the reference any more. Formats: SURVEY.md Appendix A.
"""
import gzip
import os
import subprocess
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
REF = os.path.join(ROOT, "tests", "golden", "tables")  # libriichi's data files, for the check
OUT = os.path.join(ROOT, "mortal_b200", "data")
FILES = {
    "shanten_suhai.bin": ("shanten_suhai.bin.gz", 9_703_885),
    "shanten_jihai.bin": ("shanten_jihai.bin.gz", 390_160),
    "agari.bin": ("agari.bin.gz", 86_058),
}


def generate_shanten_tables() -> dict:
    """name -> bytes, from tools/gen_shanten_tables.cc"""
    here = os.path.dirname(os.path.abspath(__file__))
    with tempfile.TemporaryDirectory() as tmp:
        exe = os.path.join(tmp, "gen_shanten_tables")
        subprocess.run(["g++", "-O2", "-std=c++17", "-o", exe, os.path.join(here, "gen_shanten_tables.cc")], check=True)
        a, b = os.path.join(tmp, "suhai.bin"), os.path.join(tmp, "jihai.bin")
        subprocess.run([exe, a, b], check=True)
        out = {}
        for name, path in (("shanten_suhai.bin", a), ("shanten_jihai.bin", b)):
            with open(path, "rb") as f:
                out[name] = f.read()[: FILES[name][1]]
            assert len(out[name]) == FILES[name][1]
    return out


def generate_agari_table() -> bytes:
    sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
    import gen_agari_table

    table = gen_agari_table.generate()
    raw = gen_agari_table.serialize(table)
    assert len(table) == 9_362 and len(raw) == FILES["agari.bin"][1]
    ref_path = os.path.join(REF, FILES["agari.bin"][0])
    if os.path.exists(ref_path):
        with gzip.open(ref_path, "rb") as f:
            assert gen_agari_table.parse(f.read()) == table, "agari.bin: generated table differs from the reference's data file"
    return raw


def main() -> int:
    os.makedirs(OUT, exist_ok=True)
    todo = [n for n in ("shanten_suhai.bin", "shanten_jihai.bin")
            if not (os.path.exists(os.path.join(OUT, n)) and os.path.getsize(os.path.join(OUT, n)) == FILES[n][1])]
    if todo:
        gen = generate_shanten_tables()
        for name in todo:
            ref_path = os.path.join(REF, FILES[name][0])
            if os.path.exists(ref_path):
                with gzip.open(ref_path, "rb") as f:
                    assert f.read() == gen[name], f"{name}: generated table differs from the reference's data file"
            with open(os.path.join(OUT, name), "wb") as f:
                f.write(gen[name])
            print(f"build_tables: generated {name} ({len(gen[name])} bytes)")
    raw = generate_agari_table()
    dst = os.path.join(OUT, "agari.bin")
    old = None
    if os.path.exists(dst):
        with open(dst, "rb") as f:
            old = f.read()
    if old != raw:  # also replaces a table gunzipped from the reference by an earlier build
        with open(dst, "wb") as f:
            f.write(raw)
        print(f"build_tables: generated agari.bin ({len(raw)} bytes)")
    return 0


if __name__ == "__main__":
    sys.exit(main())
