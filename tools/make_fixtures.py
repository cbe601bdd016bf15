#!/usr/bin/env python
"""Derive the robot descriptions used by tests and bench.py from the reference's URDF fixtures.

The reference's test URDFs (RigidBodyDynamics.jl test/urdf/*.urdf) are stored gzip-compressed under tests/golden/urdf/.
This script reads them with ``read_urdf`` (only the fields the reference's parser reads: link inertials, joint type /
parent / child / origin / axis, in document order) and writes them as JSON robot descriptions to
``rigidbodydynamics/jl_b200/models/``.  ``tests/test_urdf.py`` checks that parsing the original URDF and loading the JSON
give the same Mechanism.

    python tools/make_fixtures.py
"""
import gzip
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from rigidbodydynamics.jl_b200.urdf import read_urdf  # noqa: E402

SRC = os.path.join(ROOT, "tests", "golden", "urdf")
DST = os.path.join(ROOT, "rigidbodydynamics", "jl_b200", "models")

if __name__ == "__main__":
    os.makedirs(DST, exist_ok=True)
    for name in ("atlas", "valkyrie"):
        with gzip.open(os.path.join(SRC, name + ".urdf.gz")) as f:
            d = read_urdf(f)
        d["source"] = f"derived from RigidBodyDynamics.jl test/urdf/{name}.urdf by tools/make_fixtures.py"
        with open(os.path.join(DST, name + ".json"), "w") as f:
            json.dump(d, f, separators=(",", ":"))
        print(name, len(d["links"]), "links", len(d["joints"]), "joints")
