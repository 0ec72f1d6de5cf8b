#!/usr/bin/env python
"""Error of the int8-slice (Ozaki) product used by DF-K as a function of the slice count, in exact integer arithmetic.

Mirrors i8gemm.cuh: every row x is scaled by 2^(6-e) (|x| 2^(6-e) < 64, e from frexp of the row maximum) and cut into signed
slices q_s = rint(r_s), r_{s+1} = 128 (r_s - q_s); the product keeps the slice pairs with k + l < ns, each accumulated
exactly (int32 registers on the GPU, int64 here) and weighted 2^(ea + eb - 12 - 7 (k + l)).  Prints max |C_sliced - C| / max |C| for
random rows with a chosen dynamic range, for a contraction length K — the quantity behind "7 slices -> 4e-13 on C60" and the
question whether 6 slices would still meet the 1e-9 bar (DESIGN.md §7 item 2a).
usage: python tools/slice_error_model.py [K=65536] [rows=24] [decades=6]"""
import sys
import numpy as np


def split(x, ns):
    mx = np.abs(x).max(axis=1)
    e = np.where(mx > 0, np.frexp(mx)[1], 0)
    r = x * np.ldexp(1.0, 6 - e)[:, None]
    q = []
    for _ in range(ns):
        qs = np.rint(r)
        q.append(qs.astype(np.int64))
        r = (r - qs) * 128.0
    return q, e


def sliced_product(a, b, ns):
    qa, ea = split(a, ns)
    qb, eb = split(b, ns)
    c = np.zeros((a.shape[0], b.shape[0]), dtype=np.longdouble)
    for g in range(ns - 1, -1, -1):                      # smallest weight first, like the epilogue
        acc = np.zeros((a.shape[0], b.shape[0]), dtype=np.int64)
        for k in range(g + 1):
            acc += qa[k] @ qb[g - k].T
        c += acc.astype(np.longdouble) * np.longdouble(2.0) ** (-12 - 7 * g)
    return (c * np.ldexp(1.0, ea)[:, None].astype(np.longdouble) * np.ldexp(1.0, eb)[None, :].astype(np.longdouble))


if __name__ == '__main__':
    K = int(sys.argv[1]) if len(sys.argv) > 1 else 65536
    rows = int(sys.argv[2]) if len(sys.argv) > 2 else 24
    decades = float(sys.argv[3]) if len(sys.argv) > 3 else 6.0
    rng = np.random.RandomState(0)
    # entries with a wide dynamic range inside every row (like cderi-derived rows: a few large, most small)
    a = rng.standard_normal((rows, K)) * 10.0 ** (-decades * rng.random_sample((rows, K)))
    b = rng.standard_normal((rows, K)) * 10.0 ** (-decades * rng.random_sample((rows, K)))
    exact = a.astype(np.longdouble) @ b.astype(np.longdouble).T
    scale = np.abs(exact).max()
    print('K = %d, %d x %d outputs, max|C| = %.3e' % (K, rows, rows, float(scale)))
    for ns in (5, 6, 7, 8):
        err = np.abs(sliced_product(a, b, ns) - exact).max()
        print('  ns = %d  (%2d slice GEMMs)   max abs err / max|C| = %.2e' % (ns, ns * (ns + 1) // 2, float(err / scale)))
    print('  fp64 dot (numpy)              max abs err / max|C| = %.2e' % float(np.abs((a @ b.T).astype(np.longdouble) - exact).max() / scale))
