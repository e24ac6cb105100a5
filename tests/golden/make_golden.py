#!/usr/bin/env python3
"""Extract the reference's own known-answer vectors into JSON fixtures.

Usage: make_golden.py <path to the lewton source tree>.  The JSON files it writes
are committed and are what the tests read.  Nothing here is executed at test time.

Sources (all literal test data of the reference's own unit tests):
  * src/imdct_test.rs:11-981   IMDCT_{INPUT,OUTPUT}_TEST_ARR_{1,2,3}
  * src/header_cached.rs:117-125  bitreverse table for blocksize 8
  * src/audio.rs:294-340       low/high neighbour cases
  * src/audio.rs:369-389       render_point cases
  * src/audio.rs:437-501       FLOOR1_INVERSE_DB_TABLE (Vorbis I spec 10.1)
"""
import json
import os
import re
import sys

REF = sys.argv[1] if len(sys.argv) == 2 else None
HERE = os.path.dirname(os.path.abspath(__file__))


def read(rel):
    with open(os.path.join(REF, rel)) as f:
        return f.read()


def float_arrays(src):
    out = {}
    for m in re.finditer(r"pub static (\w+)\s*:\[f32; (\d+)\]\s*=\s*\[(.*?)\];", src, re.S):
        name, cnt, body = m.group(1), int(m.group(2)), m.group(3)
        vals = [v.strip() for v in body.replace("\n", " ").split(",") if v.strip()]
        assert len(vals) == cnt, (name, len(vals), cnt)
        out[name] = vals          # keep the decimal strings: parsed to f32 by the consumer
    return out


def main():
    if REF is None:
        sys.exit("usage: make_golden.py <path to the lewton source tree>")
    kat = float_arrays(read("src/imdct_test.rs"))
    assert set(kat) == {f"IMDCT_{d}_TEST_ARR_{i}" for d in ("INPUT", "OUTPUT") for i in (1, 2, 3)}, kat.keys()
    with open(os.path.join(HERE, "imdct_kat.json"), "w") as f:
        json.dump({"source": "lewton src/imdct_test.rs:11-981",
                   "note": "decimal strings; parse as float32. ARR_1 is the only vector the "
                           "reference's tests use (eps 5e-5, imdct.rs:831-847); ARR_2/ARR_3 are "
                           "dead data (5e-5 / 5e-4 usable, SURVEY.md section 4).",
                   "arrays": kat}, f, indent=0)

    hc = read("src/header_cached.rs")
    m = re.search(r"let cmp_arr = &\[(.*?)\];", hc, re.S)
    bitrev8 = [int(v) for v in m.group(1).replace("\n", " ").split(",") if v.strip()]
    assert len(bitrev8) == 32

    au = read("src/audio.rs")
    rp = [[int(x) for x in m.groups()] for m in re.finditer(
        r"assert_eq!\(render_point\((\d+), (\d+), (\d+), (\d+), (\d+)\), (\d+)\);", au)]
    assert len(rp) == 17
    nb = []
    # (kind, vector literal name, index, (idx, value))
    vec_simple = [1, 4, 2, 3, 6, 5]
    vec_ex = [int(v) for v in re.search(
        r"let v = \[(0, 128, 12.*?)\];", au, re.S).group(1).replace("\n", " ").split(",")]
    assert len(vec_ex) == 19
    for m in re.finditer(r"assert_eq!\((low|high)_neighbor\(&v, (\d+)\), \((\d+), (\d+)\)\);", au):
        kind, x, ri, rv = m.group(1), int(m.group(2)), int(m.group(3)), int(m.group(4))
        # the first 4+3 asserts use the 6-element vector, the rest the 19-element one
        vec = vec_simple if len(nb) < 8 else vec_ex
        nb.append({"kind": kind, "v": vec, "x": x, "idx": ri, "val": rv})
    assert len(nb) == 8 + 17, len(nb)
    tab = re.search(r"static FLOOR1_INVERSE_DB_TABLE :&\[f32\] = &\[(.*?)\];", au, re.S).group(1)
    db = [v.strip() for v in tab.replace("\n", " ").split(",") if v.strip()]
    assert len(db) == 256
    with open(os.path.join(HERE, "floor1_kat.json"), "w") as f:
        json.dump({"source": "lewton src/audio.rs:294-340,369-389,437-501; src/header_cached.rs:117-125",
                   "bitrev_bs8": bitrev8, "render_point": rp, "neighbors": nb,
                   "inverse_db_table": db}, f, indent=0)
    print("wrote imdct_kat.json, floor1_kat.json")


if __name__ == "__main__":
    main()
