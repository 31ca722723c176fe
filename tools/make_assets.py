"""Convert the reference's example OBJ input into a compact binary fixture.

Run with a checkout of the reference (ekzhang/rpt) at hand:

    RPT_REFERENCE=/path/to/rpt python tools/make_assets.py

teapot.obj (examples/teapot.rs:16) is parsed with rpt_b200.api.parse_obj -- the mirror
of src/io.rs:27-73 -- and stored as an (n, 18) float64 triangle array
(v1,v2,v3,n1,n2,n3 per row), the exact input Mesh::new receives in the reference.

pegasus.obj (examples/pegasus.zip, examples/pegasus.rs:18-32: 50 059 vertices, 100 138 faces, every
corner `f a//a`) is the scanned statue SURVEY 8(d) names as the offline stand-in for the Stanford
dragon that examples/dragon.rs:11-14 downloads.  It is stored indexed (vertices, vertex normals, faces:
float64 / int32, exactly the parsed values); rpt_b200.scenes.pegasus_proxy subdivides it to 801 104
triangles at load time.
"""
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from rpt_b200.api import parse_obj  # noqa: E402

REF = os.environ.get("RPT_REFERENCE", "")


def pegasus():
    import zipfile

    text = zipfile.ZipFile(os.path.join(REF, "examples", "pegasus.zip")).read("pegasus.obj").decode()
    v, vn, f = [], [], []
    for line in text.splitlines():
        tok = line.split()
        if not tok or tok[0].startswith("#"):
            continue
        if tok[0] == "v":
            v.append([float(x) for x in tok[1:4]])
        elif tok[0] == "vn":
            vn.append([float(x) for x in tok[1:4]])
        elif tok[0] == "f":
            corners = [c.split("/") for c in tok[1:]]
            assert len(corners) == 3 and all(c[0] == c[2] and c[1] == "" for c in corners), line
            f.append([int(c[0]) - 1 for c in corners])
    v, vn, f = np.array(v, np.float64), np.array(vn, np.float64), np.array(f, np.int32)
    assert len(v) == len(vn)
    # cross-check against the mirror of load_obj on the same text (the triangles Mesh::new would get)
    import io

    tris = parse_obj(io.StringIO(text))
    assert tris.shape == (len(f), 18)
    assert np.array_equal(tris[:, 0:9].reshape(-1, 3, 3), v[f]) and np.array_equal(tris[:, 9:18].reshape(-1, 3, 3), vn[f])
    out = os.path.join(ROOT, "rpt_b200", "assets", "pegasus_indexed.npz")
    np.savez_compressed(out, verts=v, norms=vn, faces=f)
    print(out, v.shape, f.shape, os.path.getsize(out), "bytes")


def main():
    pegasus()
    with open(os.path.join(REF, "examples", "teapot.obj")) as f:
        tris = parse_obj(f)
    out = os.path.join(ROOT, "rpt_b200", "assets", "teapot_tris.npz")
    np.savez_compressed(out, tris=tris)
    print(out, tris.shape, os.path.getsize(out), "bytes")


if __name__ == "__main__":
    main()
