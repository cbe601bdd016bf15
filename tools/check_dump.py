#!/usr/bin/env python
"""Accuracy of two `bench.py --dump-outputs` v̇ dumps (e.g. two builds) against the fp64 oracle on the same dumped columns.

Recomputes bench.py's inputs (make_inputs, PCG64 seed 1, at the batch the dumps were taken from), picks the dumped columns the
way bench.py does, runs the oracle's forward dynamics in fp64 on the fp32-rounded inputs the kernels saw, and prints one JSON
line: per dump the max and 99.9th-percentile relative error (|v̇ - v̇_ref| / max(1, |v̇_ref|_inf) per column), and the max relative
difference between the two dumps.
    python tools/check_dump.py DIR_A DIR_B [--batch B]      (default 2^20)"""
import argparse
import json
import os
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import rigidbodydynamics.jl_b200 as rbd  # noqa: E402
from bench import make_inputs  # noqa: E402
from oracle import Oracle  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("a")
    ap.add_argument("b")
    ap.add_argument("--batch", type=int, default=1 << 20)
    args = ap.parse_args()
    va, vb = (np.load(os.path.join(d, "vd.npy")).astype(np.float64) for d in (args.a, args.b))
    B, n = args.batch, va.shape[1]
    cols = np.arange(B) if n == B else np.sort(np.random.Generator(np.random.PCG64(0)).choice(B, n, replace=False))
    mech = rbd.load_model("atlas", floating=True)
    q, v, tau = make_inputs(mech, B, 1)
    q, v, tau = (x[:, cols].astype(np.float32).astype(np.float64) for x in (q, v, tau))
    ref = Oracle(mech.flatten()).dynamics(q, v, tau, nthreads=os.cpu_count() or 1)
    scale = np.maximum(1.0, np.abs(ref).max(0))
    out = {"columns": int(n)}
    for k, vd in (("a", va), ("b", vb)):
        err = np.abs(vd - ref).max(0) / scale
        out[k] = {"dir": getattr(args, k), "max_rel_err": float(err.max()), "p999_rel_err": float(np.quantile(err, 0.999))}
    out["max_rel_diff_a_b"] = float((np.abs(va - vb).max(0) / np.maximum(1.0, np.abs(va).max(0))).max())
    print(json.dumps(out))


if __name__ == "__main__":
    main()
