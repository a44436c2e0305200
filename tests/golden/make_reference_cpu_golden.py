"""Records what the reference's own CPU code (oracle/_ref/libsamplenet_ref.so, built by oracle/Makefile from the reference
sources: chamfer_distance.cpp, approxmatch.cpp) computes on the seeded inputs of tests/test_oracle_pinning.py and
tests/test_gpu_parity.py, so that those comparisons run without the reference tree.

    python tests/golden/make_reference_cpu_golden.py        (no GPU needed; needs oracle/_ref)
"""
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))

from oracle import oracle  # noqa: E402

CHAMFER_CASES = [(1, 1, 1), (2, 64, 1024), (3, 37, 129), (2, 513, 511), (1, 1024, 64), (4, 5, 3), (2, 33, 4099), (1, 6000, 70)]
CHAMFER_BWD_CASES = CHAMFER_CASES[:6]
EMD_PIN_CASES = [(64, 64), (96, 32), (40, 120)]
EMD_ASSIGN_CASES = [(64, 64), (96, 32), (40, 120), (77, 77), (300, 300)]


def chamfer_inputs(b, n, m):
    """Two clouds with exact ties (duplicated points), as in the tests."""
    r = np.random.default_rng(b * 1000 + n + m)
    a = r.standard_normal((b, n, 3)).astype(np.float32)
    c = r.standard_normal((b, m, 3)).astype(np.float32)
    if n > 4:
        a[:, 3] = a[:, 1]
    if m > 4:
        c[:, 4] = c[:, 0]
    return r, a, c


def main():
    assert oracle.have_ref(), "oracle/_ref/libsamplenet_ref.so is not built"
    out = {}
    for b, n, m in CHAMFER_CASES:
        r, a, c = chamfer_inputs(b, n, m)
        key = "chamfer_%d_%d_%d_" % (b, n, m)
        rd1, ri1, rd2, ri2 = oracle.ref_chamfer_forward(a, c)
        out.update({key + "d1": rd1, key + "i1": ri1, key + "d2": rd2, key + "i2": ri2})
        if (b, n, m) in CHAMFER_BWD_CASES:
            g1 = r.standard_normal((b, n)).astype(np.float32)
            g2 = r.standard_normal((b, m)).astype(np.float32)
            out[key + "gx1"], out[key + "gx2"] = oracle.ref_chamfer_backward(a, c, g1, ri1, g2, ri2)
    for n, m in EMD_PIN_CASES:   # tests/test_oracle_pinning.py::test_emd_oracle_vs_reference_cpu
        r = np.random.default_rng(n * 7 + m)
        a = r.random((2, n, 3)).astype(np.float32)
        c = r.random((2, m, 3)).astype(np.float32)
        key = "emd_%d_%d_" % (n, m)
        rmt = oracle.ref_approxmatch_cpu(a, c)   # (b, n, m)
        out[key + "match"] = rmt
        out[key + "cost"] = oracle.ref_matchcost_cpu(a, c, rmt)
        mt = oracle.approx_match(a, c)           # the oracle's (b, m, n) match as the input of the reference gradient
        out[key + "grad2"] = oracle.ref_matchcostgrad_cpu(a, c, np.ascontiguousarray(mt.transpose(0, 2, 1)))
    for n, m in EMD_ASSIGN_CASES:   # tests/test_gpu_parity.py::test_emd_exact_mode_bitexact_vs_oracle
        r = np.random.default_rng(n * 13 + m)
        a = r.random((3, n, 3)).astype(np.float32)
        c = r.random((3, m, 3)).astype(np.float32)
        out["emd_assign_%d_%d" % (n, m)] = oracle.ref_approxmatch_cpu(a, c).transpose(0, 2, 1).argmax(axis=2).astype(np.int32)
    path = os.path.join(HERE, "reference_cpu.npz")
    np.savez_compressed(path, **out)
    print(path, os.path.getsize(path), "bytes,", len(out), "arrays")


if __name__ == "__main__":
    main()
