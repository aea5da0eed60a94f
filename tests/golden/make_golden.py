"""Generates the committed oracle fixtures tests/golden/*.npz + golden_als.json.

There are no golden vectors in the reference (SURVEY.md 8c) and it cannot be built here, so these
fixtures freeze the outputs of oracle/buffalo_oracle.c (itself cross-checked against the NumPy fp64
restatement) at small sizes.  The CUDA parity tests replay them through the C ABI on the GPU box,
where neither the reference checkout nor a working gcc is required.

Run from the repo root:  python tests/golden/make_golden.py
"""
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
import oracle  # noqa: E402
from tests.helpers import init_factors, make_csr, transpose_csr  # noqa: E402

HERE = os.path.dirname(os.path.abspath(__file__))

CASES = [
    ("als_d20_cg", dict(d=20, optimizer="manual_cg"), 0),
    ("als_d20_cg_item", dict(d=20, optimizer="manual_cg", adaptive_reg=True), 1),
    ("als_d32_llt", dict(d=32, optimizer="llt"), 0),
    ("als_d5_ldlt_item", dict(d=5, optimizer="ldlt"), 1),
    ("als_d100_ialspp7", dict(d=100, optimizer="ialspp", block_size=7), 0),
    ("als_d128_ialspp", dict(d=128, optimizer="manual_cg"), 0),
    ("als_d128_ialspp_item", dict(d=128, optimizer="manual_cg"), 1),
    ("als_d256_ialspp", dict(d=256, optimizer="llt"), 1),
]


def main():
    meta = {"cases": []}
    U, I, nnz = 400, 250, 9000
    for name, o, axis in CASES:
        d = o["d"]
        opt = dict(num_workers=1, compute_loss_on_training=True, alpha=8.0, reg_u=0.1, reg_i=0.1, block_size=32,
                   adaptive_reg=False, num_cg_max_iters=3, eps=1e-10, cg_tolerance=1e-10)
        opt.update(o)
        indptr, keys, vals, _ = make_csr(U, I, nnz, seed=len(name), empty_rows=7)
        if axis == 1:
            indptr, keys, vals = transpose_csr(indptr, keys, vals, U, I)
        # signed factors of moderate size (a mid-training state).  All-positive factors (e.g. the very first
        # item pass after the reference's abs(N(0,1/d^2)) init) make G = Y^T Y numerically rank-1: there the fp32
        # oracle and an fp64 restatement already differ by 1e-2..1e-1 (DESIGN.md "fp32 conditioning"), so such
        # states cannot pin anything to 1e-3.
        P = init_factors(U, d, d, 11, scale=0.1, signed=True)
        Q = init_factors(I, d, d, 12, scale=0.1, signed=True)
        orc = oracle.OracleALS()
        orc.init(opt)
        P1, Q1 = P.copy(), Q.copy()
        orc.initialize_model(P1, Q1)
        orc.precompute(axis)
        rows = U if axis == 0 else I
        nume, deno = orc.partial_update(0, rows, indptr, keys, vals, axis)
        X = P1 if axis == 0 else Q1
        np.savez_compressed(os.path.join(HERE, name + ".npz"), P=P, Q=Q, indptr=indptr, keys=keys, vals=vals,
                            X=X, nume=nume, deno=deno)
        meta["cases"].append({"file": name + ".npz", "opt": opt, "axis": axis})
    json.dump(meta, open(os.path.join(HERE, "golden_als.json"), "w"), indent=1)


if __name__ == "__main__":
    main()
