"""numpy model of the int8-slice DF-K engine (pyscf_b200/csrc/i8gemm.cuh), precise enough to predict its output bit for bit,
and an exact reference for C = A B^T.

The engine's arithmetic is deterministic wherever it is exact: the slices are integers, the slice-pair group sums are exact
int32 sums (any order), and the fp64 fold g = NS-1 ... 0 with weights 2^(-12-7g) followed by the exponent scaling is a fixed
sequence of roundings.  Only the fp64 reductions that join several K ranges (stage 2, atomicAdd) and the float32 row norms
behind the exponent bound of Y (atomicAdd) depend on the order of execution; the model bounds the first and takes the second
from the kernel when a test needs bit-exact Y digits.

Digit conventions (row exponent e: |x| < 2^e, the row's largest element has frexp exponent e; a zero row has e = 0):
  rint       x 2^(6-e) = sum_s q_s 2^(-7s) + tail, q_s = rint of the running remainder (ties to even), |q_s| <= 64
             (split_rows_kernel, split_long_kernel, split_packed_kernel with ns = 8)
  mantissa   N = rint(x 2^(6-e+7(ns-1))), q_0 = N >> 7(ns-1) (signed, |q_0| <= 64), q_s = (N >> 7(ns-1-s)) & 127 for s >= 1
             (split_packed_kernel with ns <= 7, both the NS7 and the generic path)
  yfused     the rint digits of Y 2^(6-Ey), cut in the stage-1 epilogue with the 1.5 2^52 trick: the digit is the low byte
             of the rounded value (it wraps when |Y| >= 2^Ey, i.e. when Ey is not a bound)
"""
from fractions import Fraction

import numpy as np

BM, BN, BK = 128, 32, 128
INT32_MAX = 2 ** 31 - 1


def pad_to(n, m):
    return (n + m - 1) // m * m


def stack_rows(n):
    """Rows of a slice stack: a multiple of 256 (both BM and BN)."""
    return pad_to(n, 256)


# ------------------------------------------------------------------------------------------------- exponents
def frexp_exp(v):
    """Biased exponent - 1022 of |v| (v != 0): the frexp exponent of a normal number, -1022 for every subnormal."""
    bits = np.abs(np.asarray(v, dtype=np.float64)).view(np.int64)
    return ((bits >> 52) & 0x7ff).astype(np.int64) - 1022


def row_exponents(X):
    """frexp exponent of each row's largest |element| (split_rows, split_long), 0 for a zero row."""
    mx = np.abs(X).max(axis=1) if X.shape[1] else np.zeros(X.shape[0])
    return maxima_exponents(mx)


def maxima_exponents(mx):
    """Row exponents from given row maxima (split_rows_premax)."""
    e = np.frexp(np.asarray(mx, dtype=np.float64))[1].astype(np.int64)
    return np.where(np.asarray(mx) > 0, e, 0)


def unpack_rows(cderi, nao):
    """Unpacked tensor rows (P, a) -> A_P[a][:] of packed rows cderi[P][a(a+1)/2 + b], a >= b: [nr*nao][nao]."""
    nr = cderi.shape[0]
    i, j = np.tril_indices(nao)
    A = np.zeros((nr, nao, nao))
    A[:, i, j] = cderi
    A[:, j, i] = cderi
    return A.reshape(nr * nao, nao)


def packed_rowexp(cderi, nao):
    """packed_rowexp_kernel: max over the unpacked row of frexp_exp of its non-zero elements; EXP_NONE (no non-zero) -> 0."""
    X = unpack_rows(cderi, nao)
    e = np.where(X != 0, frexp_exp(np.where(X != 0, X, 1.0)), -(1 << 40))
    e = e.max(axis=1) if X.shape[1] else np.full(X.shape[0], -(1 << 40))
    return np.where(e == -(1 << 40), 0, e)


# ------------------------------------------------------------------------------------------------- digits
def digits_rint(X, E, ns):
    """[ns][R][K] int8 balanced digits of the rows of X scaled by 2^(6-E)."""
    rr = np.ldexp(X, (6 - np.asarray(E))[:, None].astype(np.int32))
    q = np.empty((ns,) + X.shape, dtype=np.int8)
    for s in range(ns):
        qv = np.rint(rr)
        q[s] = qv.astype(np.int64).astype(np.int8)
        rr = (rr - qv) * 128.0
    return q


def digits_mantissa(X, E, ns):
    """[ns][R][K] int8 digits of N = rint(x 2^(6-E+7(ns-1))): signed top digit, the others 0..127."""
    N = np.rint(np.ldexp(X, (6 - np.asarray(E) + 7 * (ns - 1))[:, None].astype(np.int32))).astype(np.int64)
    q = np.empty((ns,) + X.shape, dtype=np.int8)
    for s in range(ns):
        sh = 7 * (ns - 1 - s)
        d = (N >> sh) if s == 0 else ((N >> sh) & 127)
        q[s] = d.astype(np.int8)
    return q


def digits_yfused(R, ns):
    """[ns][...] int8 digits of already scaled values R (the stage-1 epilogue): low byte of rint(r) (wraps past 127)."""
    r = np.array(R, dtype=np.float64)
    q = np.empty((ns,) + r.shape, dtype=np.int8)
    for s in range(ns):
        qv = (r + 6755399441055744.0) - 6755399441055744.0
        q[s] = qv.astype(np.int64).astype(np.int8)
        r = (r - qv) * 128.0
    return q


def reconstruct(q, E):
    """The value a digit stack represents: 2^E sum_s q_s 2^(-6-7s) (exact in fp64 for ns <= 7 balanced digits)."""
    ns = q.shape[0]
    v = sum(q[s].astype(np.float64) * 2.0 ** (-6 - 7 * s) for s in range(ns))
    return np.ldexp(v, np.asarray(E)[:, None].astype(np.int32))


# ------------------------------------------------------------------------------------------------- stacks
class Stack:
    """[ns][Rp][Kp] int8 slices + E[Rp], pads zero; dmax = largest |digit| the convention allows."""

    def __init__(self, q, E, dmax=64):
        ns, R, K = q.shape
        self.ns, self.R, self.K = ns, R, K
        self.Rp, self.Kp = stack_rows(R), pad_to(K, BK)
        self.q = np.zeros((ns, self.Rp, self.Kp), dtype=np.int8)
        self.q[:, :R, :K] = q
        self.E = np.zeros(self.Rp, dtype=np.int64)
        self.E[:R] = E
        self.dmax = dmax


def slice_rows(X, ns, rowmax=None):
    """split_rows / split_long / split_rows_premax (given row maxima)."""
    E = row_exponents(X) if rowmax is None else maxima_exponents(rowmax)
    return Stack(digits_rint(X, E, ns), E)


def slice_packed(cderi, nao, ns):
    """packed_rowexp + split_packed: (stack of the nr*nao unpacked rows, rowexp[nr][nao])."""
    E = packed_rowexp(cderi, nao)
    X = unpack_rows(cderi, nao)
    if ns <= 7:
        return Stack(digits_mantissa(X, E, ns), E, dmax=127), E.reshape(cderi.shape[0], nao)
    return Stack(digits_rint(X, E, ns), E), E.reshape(cderi.shape[0], nao)


# ------------------------------------------------------------------------------------------------- GEMM
def group_sums(qa, qb, wrap=False):
    """G[g] = sum_{k+l=g} qa[k] qb[l]^T, exact.  The int8 products and their sums stay far below 2^53, so fp64 matrix
    products are exact here.  A sum outside int32 raises OverflowError (the kernel would wrap it); wrap=True returns the
    wrapped value instead."""
    ns = qa.shape[0]
    if qa.shape[-1] * 127 * 127 * ns >= 2 ** 53:
        raise ValueError('K too long for the exact fp64 model of the group sums')
    A = qa.astype(np.float64)
    B = qb.astype(np.float64)
    G = np.zeros((ns, qa.shape[1], qb.shape[1]), dtype=np.int64)
    for k in range(ns):
        for l in range(ns - k):
            G[k + l] += (A[k] @ B[l].T).astype(np.int64)
    if G.max(initial=0) > INT32_MAX or G.min(initial=0) < -2 ** 31:
        if not wrap:
            raise OverflowError('slice-pair group sum outside int32')
        G = ((G + 2 ** 31) % 2 ** 32) - 2 ** 31
    return G


def fold(G):
    """fp64 fold of the kernel: g = NS-1 ... 0, acc += G_g 2^(-12-7g)."""
    ns = G.shape[0]
    acc = np.zeros(G.shape[1:])
    for g in range(ns - 1, -1, -1):
        acc = acc + G[g].astype(np.float64) * 2.0 ** (-12 - 7 * g)
    return acc


def product(A, B, a_row0=0, m=None, k0=0, k1=None, wrap=False):
    """One work item range of the kernel: rows [a_row0, a_row0+m) of A times all rows of B over K columns [k0, k1),
    folded and scaled: the fp64 value the epilogue stores (before any scatter / accumulation)."""
    m = A.R - a_row0 if m is None else m
    k1 = A.Kp if k1 is None else k1
    qa = A.q[:, a_row0:a_row0 + m, k0:k1]
    qb = B.q[:, :B.R, k0:k1]
    acc = fold(group_sums(qa, qb, wrap=wrap))
    with np.errstate(over='ignore'):
        return acc, np.ldexp(acc, (A.E[a_row0:a_row0 + m][:, None] + B.E[:B.R][None, :]).astype(np.int32))


def stage1(A, B, a_row0=0, m=None, inner=0):
    """gemm_ar plain epilogue: (C, rowmax).  inner > 0: C[m % inner][(m // inner) N + n] (transposed scatter)."""
    m = A.R - a_row0 if m is None else m
    _, V = product(A, B, a_row0, m)
    N = B.R
    if inner <= 0:
        C = V
        rowmax = np.abs(V).max(axis=1)
    else:
        nblk = (m + inner - 1) // inner
        Vp = np.zeros((nblk * inner, N))
        Vp[:m] = V
        C = Vp.reshape(nblk, inner, N).transpose(1, 0, 2).reshape(inner, nblk * N)
        rowmax = np.abs(Vp).reshape(nblk, inner, N).max(axis=(0, 2))
    return C, rowmax


def stage1_y(A, B, Ey, a_row0, m, inner, y_ncolp):
    """gemm_ar with the fused Y epilogue: the Y stack (rows inner, columns (m // inner) y_ncolp) with exponents Ey."""
    ns = A.ns
    acc, _ = product(A, B, a_row0, m)
    Eb = np.zeros(y_ncolp, dtype=np.int64)
    Eb[:min(B.R, y_ncolp)] = B.E[:min(B.R, y_ncolp)]
    accp = np.zeros((m, y_ncolp))
    accp[:, :B.R] = acc
    rows = np.arange(m)
    esc = A.E[a_row0 + rows] + 6 - np.asarray(Ey)[rows % inner]
    R = np.ldexp(accp, (esc[:, None] + Eb[None, :]).astype(np.int32))
    d = digits_yfused(R, ns)                                    # [ns][m][y_ncolp]
    nblk = m // inner
    q = d.reshape(ns, nblk, inner, y_ncolp).transpose(0, 2, 1, 3).reshape(ns, inner, nblk * y_ncolp)
    return Stack(q, Ey)


def stage2(A, B, symmetric=False, kb_per=None, exact_ranges=False):
    """gemm_ar_acc from C = 0 with K ranges of kb_per blocks.  One range: the exact result of the kernel.  Several: the
    ranges are summed here in order and bounded by ranges_bound (the kernel adds them with fp64 atomics in any order).
    Returns (C, list of the per-range values)."""
    nkb = A.Kp // BK
    kb_per = nkb if not kb_per else min(kb_per, nkb)
    parts = []
    for kb0 in range(0, nkb, kb_per):
        parts.append(product(A, B, 0, A.R, kb0 * BK, min(nkb, kb0 + kb_per) * BK)[1])
    C = parts[0].copy()
    for p in parts[1:]:
        C = C + p
    if symmetric:
        C = np.triu(C)
        parts = [np.triu(p) for p in parts]
    return C, parts


def ranges_bound(parts):
    """Bound on the difference between two summation orders of the per-range values (fp64 re-association)."""
    if len(parts) == 1:
        return np.zeros_like(parts[0])
    s = sum(np.abs(p) for p in parts)
    return 2.0 * (len(parts) - 1) * 2.0 ** -53 * s


def int32_ok(ns, k, dmax_a, dmax_b):
    """The bound gemm_ar / gemm_ar_acc enforce per K range: ns pairs of k products of |digits| <= dmax_a, dmax_b."""
    return ns * k * dmax_a * dmax_b <= INT32_MAX


# ------------------------------------------------------------------------------------------------- error bounds
def tail_bound(ns):
    """Largest |representation error| of one digit stack, in units of 2^E: half of the last digit's weight."""
    return 2.0 ** (-7 * ns)


def product_bound(ns, K, Ea, Eb, dmax_a=64, dmax_b=64):
    """Bound on |model - exact| of C = A B^T, per element [len(Ea)][len(Eb)], for operands sliced with row exponents Ea, Eb:
    representation tails of both operands, the slice pairs k + l >= ns that are never formed, and the fp64 fold."""
    w = lambda g: 2.0 ** (-12 - 7 * g)
    dropped = sum((2 * ns - 1 - g) * w(g) for g in range(ns, 2 * ns - 1)) * dmax_a * dmax_b
    size = sum((g + 1) * w(g) for g in range(ns)) * dmax_a * dmax_b       # |acc| per K term
    per_term = 2 * tail_bound(ns) * (1 + tail_bound(ns)) + dropped + (ns + 1) * 2.0 ** -53 * size
    with np.errstate(over='ignore'):
        scale = np.ldexp(1.0, (np.asarray(Ea)[:, None] + np.asarray(Eb)[None, :]).astype(np.int32))
    return K * per_term * scale + 2.0 ** -1073


# ------------------------------------------------------------------------------------------------- exact reference
def _int_rows(X):
    """X[i] = I[i] 2^s[i] exactly, I a row of Python ints."""
    X = np.asarray(X, dtype=np.float64)
    m, e = np.frexp(X)
    mi = np.ldexp(m, 53).astype(np.int64)
    ee = e.astype(np.int64) - 53
    I = np.empty(X.shape, dtype=object)
    s = np.zeros(X.shape[0], dtype=np.int64)
    for i in range(X.shape[0]):
        nz = mi[i] != 0
        s[i] = ee[i][nz].min() if nz.any() else 0
        I[i] = [int(a) << int(b - s[i]) if a else 0 for a, b in zip(mi[i], ee[i])]
    return I, s


def _to_float(n, s):
    """n 2^s rounded once to the nearest double (Python int conversion and true division round correctly)."""
    if n == 0:
        return 0.0
    if s >= 0:
        try:
            return float(n << s)
        except OverflowError:
            return float('inf') if n > 0 else float('-inf')
    return n / (1 << -s)


def exact_abt(A, B):
    """C = A B^T computed exactly from the fp64 inputs and rounded once per element."""
    IA, sa = _int_rows(A)
    IB, sb = _int_rows(B)
    P = IA.dot(IB.T)
    return np.array([[_to_float(int(P[i, j]), int(sa[i] + sb[j])) for j in range(P.shape[1])] for i in range(P.shape[0])])


def exact_value(X):
    """Fractions of the entries (for exact comparisons of representations)."""
    return np.vectorize(Fraction, otypes=[object])(X)
