"""The 4-center Rys kernels class by class against high-precision integrals, and the Rys tables they all draw from.

* Rys quadrature (b200jk_rys_test): the rule rys_root evaluates, for n = 1..9 at every interval edge and midpoint of the
  table, at 0, 1e-300, a subnormal, around the switch to the Hermite branch at x = 100 and far beyond.  Moments
  sum_r w_r u_r^k against F_k(x) from mpmath, roots and weights against an mpmath Golub-Welsch, continuity at every edge,
  and on the GPU the device kernel against the emulation.
* Integrals: unit densities through the public J/K entry point recover every (ij|kl) of the shipped kernels (K route:
  hermi = 0, D = E_jk gives K_il = (ij|kl); J route: D = E_kl + E_lk gives J_ij = 2 (ij|kl)).  Each element is compared
  with tests/eri_ref.py (McMurchie-Davidson in long double) and labelled with its class as launched and its kernel family.

Accuracy bar: |kernel - ref| <= KAPPA * eps * S, S the maximum of S_abs (sum of absolute primitive-quartet contributions)
over the shell-quartet block.  The K route of a non-symmetric density adds a symmetric and an antisymmetric part, each
carrying (ij|kl) and (ik|jl); its scale is the larger S of the two blocks.  A block whose S is exactly 0 (parity zeros of
one-centre quartets: the centres are dyadic, so P - A is exactly 0 in double precision) must come out exactly 0.
"""
import ctypes
import time

import mpmath as mp
import numpy as np
import pytest

import eri_ref as R
from pyscf_b200 import gto
from pyscf_b200 import lib as b2lib
from pyscf_b200.jk import VHFOpt

pytestmark = pytest.mark.skipif(not R.LONGDOUBLE_OK, reason=R.SKIP_REASON)

EPS = np.finfo(np.float64).eps
# Largest error / S measured over every class and case below: 57 eps on the CPU emulation ((dp|fp)) and 50 eps on one H100
# ((dp|fp)); per class in DESIGN.md §4.1.  KAPPA keeps more than a 10x margin, and KAPPA * eps = 2.3e-13 stays below 1e-12,
# so a 1e-11 relative error in any class fails.
KAPPA = 1024
BAR = KAPPA * EPS
# Only in the `far` system, blocks below FLOOR of the system's largest S are held to FLOOR * S_max instead.  Their relative
# accuracy is limited by the horizontal recurrence over pairs 17.9 bohr apart with disparate exponents (AB^k terms that
# cancel to a tiny integral): (dd|dd) of a d pair with exponents 25 and 0.1, |(ij|kl)| ~ 2e-27, comes out with error
# 3.5e-9 of S.  The floor those blocks need, measured on the emulation for all four operators, is at most 9e-14 of S_max;
# FLOOR keeps a 100x margin.  Every other system is held to the plain relative bar in every block.
FLOOR = {'far': 1e-11}

# ---------------------------------------------------------------------------------------------------------------------
# Rys tables
RYS_NMAX, RYS_NINT, RYS_H, RYS_XMAX = 9, 320, 0.3125, 100.0
TABLE_ERR = 3.6e-15      # largest absolute error of a tabulated root or weight (tools/gen_rys_tables.py self-check)


def rys_points():
    xs = [0.0, 1e-300, 5e-324, 2.5e-310, np.nextafter(RYS_XMAX, 0), RYS_XMAX, np.nextafter(RYS_XMAX, np.inf), 1e3, 1e6, 1e12]
    for iv in range(RYS_NINT):
        lo, hi = iv * RYS_H, (iv + 1) * RYS_H
        xs += [lo, np.nextafter(hi, 0), lo + RYS_H / 2]
    return np.array(sorted(set(xs)))


def rys_eval(lib, n, x):
    h = b2lib.Handle(*_tiny_tables(), libpath=lib)
    x = np.ascontiguousarray(x, dtype=np.float64)
    u = np.zeros((len(x), n))
    w = np.zeros((len(x), n))
    h.check(h.lib.b200jk_rys_test(h._h, n, len(x), b2lib.dptr(x), b2lib.dptr(u), b2lib.dptr(w)), 'b200jk_rys_test')
    h.close()
    return u, w


def _tiny_tables():
    m = gto.M(atom='H 0 0 0; H 0 0 1.4', unit='Bohr', basis='sto-3g')
    return m._atm, m._bas, m._env


def boys_mp(kmax, x):
    """F_0..F_kmax at x in mpmath (the top order from the incomplete gamma function, then downward recursion)."""
    x = mp.mpf(x)
    if x == 0:
        return [mp.mpf(1) / (2 * k + 1) for k in range(kmax + 1)]
    F = [None] * (kmax + 1)
    F[kmax] = mp.gammainc(kmax + mp.mpf(1) / 2, 0, x) / (2 * x ** (kmax + mp.mpf(1) / 2))
    e = mp.exp(-x)
    for k in range(kmax - 1, -1, -1):
        F[k] = (2 * x * F[k + 1] + e) / (2 * k + 1)
    return F


def golub_welsch(n, x):
    """n-point Gauss rule of the weight exp(-x u)/(2 sqrt(u)) on [0, 1], whose moments are F_k(x): Cholesky of the Hankel
    moment matrix, Jacobi matrix, eigen-decomposition (80 digits)."""
    with mp.workdps(80):
        mu = boys_mp(2 * n, x)
        Hm = mp.matrix(n + 1, n + 1)
        for i in range(n + 1):
            for j in range(n + 1):
                Hm[i, j] = mu[i + j]
        Rm = mp.cholesky(Hm).T
        J = mp.matrix(n, n)
        for j in range(n):
            J[j, j] = Rm[j, j + 1] / Rm[j, j] - (Rm[j - 1, j] / Rm[j - 1, j - 1] if j > 0 else 0)
            if j + 1 < n:
                J[j, j + 1] = J[j + 1, j] = Rm[j + 1, j + 1] / Rm[j, j]
        E, Q = mp.eigsy(J)
        order = sorted(range(n), key=lambda i: E[i])
        return [float(E[i]) for i in order], [float(mu[0] * Q[0, i] ** 2) for i in order]


def check_rys(lib):
    xs = rys_points()
    F = {}
    with mp.workdps(40):
        for x in xs:
            F[x] = [float(v) for v in boys_mp(2 * RYS_NMAX - 1, x)]
    worst_mom, worst_node, worst_jump = 0.0, 0.0, 0.0
    out = {}
    for n in range(1, RYS_NMAX + 1):
        u, w = rys_eval(lib, n, xs)
        out[n] = (u, w)
        assert np.all(np.isfinite(u)) and np.all(np.isfinite(w)), n
        # moments: sum_r w_r u_r^k = F_k(x), k = 0..2n-1.  Bar: the table's absolute error TABLE_ERR on every u_r and w_r
        # moves the sum by at most TABLE_ERR * sum_r (u_r^k + k w_r u_r^(k-1)); above x = 100 the rule is the scaled
        # Gauss-Hermite one and only rounding remains (2n eps relative).  Factor 4 for the evaluation itself.
        for k in range(2 * n):
            mom = (w * u ** k).sum(axis=1)
            ref = np.array([F[x][k] for x in xs])
            tab = TABLE_ERR * ((u ** k).sum(axis=1) + (k * w * u ** max(k - 1, 0)).sum(axis=1))
            tab = np.where(xs >= RYS_XMAX, 0.0, tab)
            bar = 4 * (tab + 2 * n * (k + 1) * EPS * np.abs(ref)) + 1e-300
            err = np.abs(mom - ref)
            i = int(np.argmax(err / bar))
            assert err[i] <= bar[i], 'n=%d k=%d x=%r: |sum w u^k - F_k| = %.3e, F_k = %.3e, bar %.3e' % (
                n, k, xs[i], err[i], ref[i], bar[i])
            worst_mom = max(worst_mom, float((err / bar).max()))
        # continuity: the two pieces that meet at an interval edge (and the Chebyshev and Hermite branches at x = 100)
        # agree within twice the table error
        for iv in range(1, RYS_NINT + 1):
            e = iv * RYS_H
            a, b = np.searchsorted(xs, np.nextafter(e, 0)), np.searchsorted(xs, e)
            assert xs[a] == np.nextafter(e, 0) and xs[b] == e
            jump = max(np.abs(u[a] - u[b]).max(), np.abs(w[a] - w[b]).max())
            assert jump <= 2 * TABLE_ERR + 8 * EPS, 'n=%d: jump %.3e at x=%r' % (n, jump, e)
            worst_jump = max(worst_jump, jump)
    # roots and weights against a fresh Golub-Welsch, about 50 points per n: edges, midpoints and the x = 100 switch
    rng = np.random.RandomState(5)
    for n in range(1, RYS_NMAX + 1):
        pts = np.concatenate([[0.0, 1e-300, np.nextafter(RYS_XMAX, 0), RYS_XMAX, 1e3],
                              rng.choice(xs[(xs > 0) & (xs < RYS_XMAX)], 45, replace=False)])
        u, w = rys_eval(lib, n, pts)
        for i, x in enumerate(pts):
            if x >= RYS_XMAX:
                ue, we = golub_welsch(n, x)
                tol = 16 * EPS * np.abs(ue).max() + 1e-300, 16 * EPS * np.abs(we).max()
            else:
                ue, we = golub_welsch(n, x)
                tol = 2 * TABLE_ERR, 2 * TABLE_ERR
            du, dw = np.abs(u[i] - ue).max(), np.abs(w[i] - we).max()
            assert du <= tol[0] and dw <= tol[1], 'n=%d x=%r: |du| %.3e |dw| %.3e' % (n, x, du, dw)
            worst_node = max(worst_node, du, dw)
    print('Rys: worst moment error / bar %.3f, worst root/weight error %.2e, worst jump at an edge %.2e' % (
        worst_mom, worst_node, worst_jump))
    return xs, out


def test_rys_emulated(emu_lib):
    check_rys(emu_lib)


def test_rys_rejects_bad_arguments(emu_lib):
    h = b2lib.Handle(*_tiny_tables(), libpath=emu_lib)
    x = np.array([1.0, np.nan])
    u = np.zeros(2 * 3)
    assert h.lib.b200jk_rys_test(h._h, 3, 2, b2lib.dptr(x), b2lib.dptr(u), b2lib.dptr(u.copy())) != 0
    assert h.lib.b200jk_rys_test(h._h, 10, 1, b2lib.dptr(x), b2lib.dptr(u), b2lib.dptr(u.copy())) != 0
    h.close()


@pytest.mark.gpu
def test_rys_device(emu_lib):
    xs, dev = check_rys(None)
    for n in range(1, RYS_NMAX + 1):
        ue, we = rys_eval(emu_lib, n, xs)
        u, w = dev[n]
        # FMA contraction in the Clenshaw recurrence is the only expected difference: a few ulp of the largest node/weight
        su = 16 * EPS * np.abs(ue).max(axis=1, keepdims=True) + 1e-300
        sw = 16 * EPS * np.abs(we).max(axis=1, keepdims=True) + 1e-300
        assert np.all(np.abs(u - ue) <= su) and np.all(np.abs(w - we) <= sw), n


# ---------------------------------------------------------------------------------------------------------------------
# Reference validation
def test_reference_boys_against_mpmath():
    xs = [0.0, 1e-300, 1e-12, 1e-6, 0.3] + [iv * RYS_H for iv in range(0, RYS_NINT + 1, 7)] + \
         [np.nextafter(50.0, 0), 50.0, 99.9, 100.0, 150.0, 400.0, 1e3, 3e3, 1e4]
    F = R.boys(16, np.array(xs, dtype=R.LD))
    worst = 0.0
    with mp.workdps(40):
        for i, x in enumerate(xs):
            ref = boys_mp(16, x)
            for m in range(17):
                rel = abs(mp.mpf(str(F[m, i])) - ref[m]) / ref[m]
                worst = max(worst, float(rel))
    assert worst < 2e-18, worst      # long double: eps 1.1e-19


def _prim_quartet(ls, exps, centres, omega=0.0):
    """Bare Cartesian primitive quartet (no coefficients, no s/p factors) from the reference."""
    segs = [R._Seg(l, np.array(c, dtype=R.LD), np.array([e]), np.array([1.0]), 0) for l, e, c in zip(ls, exps, centres)]
    bra, ket = R._Pair(segs[0], segs[1], 0.0), R._Pair(segs[2], segs[3], 0.0)
    fac = np.prod([float(R._SP_FAC.get(l, 1)) for l in ls])
    v, _, _ = R.quartet(bra, ket, omega)
    return v / R.LD(fac)


def _md_mpmath(ls, exps, centres, omega=0.0):
    """The same McMurchie-Davidson formulas evaluated in mpmath, one element at a time."""
    mp.mp.dps = 40
    A, B, C, D = [[mp.mpf(v) for v in c] for c in centres]
    a, b, c, d = [mp.mpf(e) for e in exps]

    def E1(i, j, PA, PB, p):
        E = {(0, 0, 0): mp.mpf(1)}
        g = lambda i_, j_, t: E.get((i_, j_, t), mp.mpf(0))
        for ii in range(i + 1):
            for jj in range(j + 1):
                if ii == jj == 0:
                    continue
                for t in range(ii + jj + 1):
                    if ii > 0:
                        E[ii, jj, t] = g(ii - 1, jj, t - 1) / (2 * p) + PA * g(ii - 1, jj, t) + (t + 1) * g(ii - 1, jj, t + 1)
                    else:
                        E[ii, jj, t] = g(ii, jj - 1, t - 1) / (2 * p) + PB * g(ii, jj - 1, t) + (t + 1) * g(ii, jj - 1, t + 1)
        return E

    def pair(X, Y, ex, ey, lx, ly):
        p = ex + ey
        P = [(ex * X[k] + ey * Y[k]) / p for k in range(3)]
        K = mp.exp(-ex * ey / p * sum((X[k] - Y[k]) ** 2 for k in range(3)))
        Es = [E1(lx, ly, P[k] - X[k], P[k] - Y[k], p) for k in range(3)]
        return p, P, K, Es

    p, P, K1, Eb = pair(A, B, a, b, ls[0], ls[1])
    q, Q, K2, Ek = pair(C, D, c, d, ls[2], ls[3])
    al = p * q / (p + q)
    pref = 2 * mp.pi ** mp.mpf(2.5) / (p * q * mp.sqrt(p + q)) * K1 * K2
    if omega > 0:
        th = mp.mpf(omega) ** 2 / (mp.mpf(omega) ** 2 + al)
        al *= th
        pref *= mp.sqrt(th)
    PQ = [P[k] - Q[k] for k in range(3)]
    L = sum(ls)
    F = boys_mp(L, al * sum(v ** 2 for v in PQ))
    Rt = {}

    def Rf(t, u, v, n):
        if (t, u, v, n) in Rt:
            return Rt[t, u, v, n]
        if t < 0 or u < 0 or v < 0:
            return mp.mpf(0)
        if t == u == v == 0:
            r = (-2 * al) ** n * F[n]
        elif t > 0:
            r = (t - 1) * Rf(t - 2, u, v, n + 1) + PQ[0] * Rf(t - 1, u, v, n + 1)
        elif u > 0:
            r = (u - 1) * Rf(t, u - 2, v, n + 1) + PQ[1] * Rf(t, u - 1, v, n + 1)
        else:
            r = (v - 1) * Rf(t, u, v - 2, n + 1) + PQ[2] * Rf(t, u, v - 1, n + 1)
        Rt[t, u, v, n] = r
        return r

    ca, cb, cc, cd = [R.cart_comps(l) for l in ls]
    Lb, Lk = ls[0] + ls[1], ls[2] + ls[3]
    hb, hk = R._herm(Lb), R._herm(Lk)
    out = np.zeros((len(ca) * len(cb), len(cc) * len(cd)))
    # T[h][cd] = sum_h' (-1)^|h'| E^cd_h' R_{h+h'}
    Ecd = [[Ek[0].get((kc[0], kd[0], t2), 0) * Ek[1].get((kc[1], kd[1], u2), 0) * Ek[2].get((kc[2], kd[2], v2), 0)
            for (t2, u2, v2) in hk] for kc in cc for kd in cd]
    T = [[sum(Ecd[j][k] * (-1) ** sum(hk[k]) * Rf(t + hk[k][0], u + hk[k][1], v + hk[k][2], 0)
              for k in range(len(hk)) if Ecd[j][k] != 0) for j in range(len(Ecd))] for (t, u, v) in hb]
    for i, (ka, kb) in enumerate([(x, y) for x in ca for y in cb]):
        Eab = [Eb[0].get((ka[0], kb[0], t), 0) * Eb[1].get((ka[1], kb[1], u), 0) * Eb[2].get((ka[2], kb[2], v), 0)
               for (t, u, v) in hb]
        for j in range(len(Ecd)):
            out[i, j] = float(pref * sum(Eab[h] * T[h][j] for h in range(len(hb)) if Eab[h] != 0))
    return out


def test_reference_ssss_closed_form():
    mp.mp.dps = 40
    A, B, C, D = (0, 0, 0), (0.5, -0.25, 1.0), (1.5, 2.0, -0.5), (-1.0, 0.75, 0.25)
    for exps, omega in (((1.3, 0.4, 7.0, 0.05), 0.0), ((1e4, 0.3, 2.0, 2.0), 0.0), ((1.3, 0.4, 7.0, 0.05), 0.35)):
        v = float(_prim_quartet((0, 0, 0, 0), exps, (A, B, C, D), omega)[0, 0])
        a, b, c, d = [mp.mpf(e) for e in exps]
        p, q = a + b, c + d
        P = [(a * A[k] + b * B[k]) / p for k in range(3)]
        Q = [(c * C[k] + d * D[k]) / q for k in range(3)]
        K = mp.exp(-a * b / p * sum((mp.mpf(A[k]) - B[k]) ** 2 for k in range(3)) -
                   c * d / q * sum((mp.mpf(C[k]) - D[k]) ** 2 for k in range(3)))
        al = p * q / (p + q)
        if omega:
            al = al * omega ** 2 / (omega ** 2 + al)
        T = al * sum((P[k] - Q[k]) ** 2 for k in range(3))
        ref = 2 * mp.pi ** 2.5 / (p * q * mp.sqrt(p + q)) * K * mp.sqrt(al / (p * q / (p + q))) * mp.sqrt(mp.pi / T) / 2 * mp.erf(mp.sqrt(T))
        assert abs(v - float(ref)) <= 4 * EPS * abs(float(ref)), (exps, omega, v, float(ref))


@pytest.mark.parametrize('ls,exps,omega', [((2, 2, 2, 2), (1.7, 0.6, 3.1, 0.35), 0.0),
                                           ((3, 2, 1, 1), (2.2, 0.8, 0.45, 5.0), 0.0),
                                           ((3, 2, 1, 1), (2.2, 0.8, 0.45, 5.0), 0.35)])
def test_reference_primitive_quartet_against_mpmath(ls, exps, omega):
    centres = ((0, 0, 0), (0.5, -0.25, 1.0), (1.5, 2.0, -0.5), (-1.0, 0.75, 0.25))
    v = _prim_quartet(ls, exps, centres, omega).astype(np.float64)
    ref = _md_mpmath(ls, exps, centres, omega)
    assert np.abs(v - ref).max() <= 8 * EPS * np.abs(ref).max(), np.abs(v - ref).max() / np.abs(ref).max()


def test_reference_c2s_matches_oracle():
    from oracle import oracle as O
    for l in range(4):
        c = np.zeros((2 * l + 1) * R.ncart(l))
        O.lib().oracle_c2s(ctypes.c_int(l), O._p(c))
        m = R.c2s_matrix(l).astype(np.float64) * float(R._SP_FAC.get(l, 1))
        assert np.abs(c.reshape(2 * l + 1, -1) - m).max() < 4 * EPS, l


def test_reference_against_oracle_and_golden():
    from oracle import oracle as O
    # dyadic centres in Bohr: one-centre parity zeros are exact zeros on both sides
    mol = gto.M(atom='He 0 0 0; Ne 0.5 1 2', unit='Bohr', basis='ccpvdz')
    ref = R.Reference(mol._atm, mol._bas, mol._env, prim_cut=0.0)
    e, s = ref.eri_cart()
    T = ref.c2s()
    es, ss = R.to_sph(e, T).astype(np.float64), R.to_sph(s, np.abs(T)).astype(np.float64)
    o = O.int2e(mol)
    ratio = block_ratio(np.abs(es - o), block_max(ss, sph_offsets(ref)), sph_offsets(ref))
    assert ratio.max() <= 1e-13, ratio.max()
    oc = O.int2e(mol, cart=True)
    offc = cart_offsets(ref)
    ratio = block_ratio(np.abs(e.astype(np.float64) - oc), block_max(s.astype(np.float64), offc), offc)
    assert ratio.max() <= 1e-13, ratio.max()
    # pyscf/gto/test/test_moleintor.py:317-320, the fingerprint tests/test_oracle_golden.py pins for the oracle
    mol = gto.M(atom='He 0 0 0; Ne 3 0 0', basis='ccpvdz')
    ref = R.Reference(mol._atm, mol._bas, mol._env, prim_cut=0.0)
    e, _ = ref.eri_cart()
    assert abs(O.fp(O.s8_pack(R.to_sph(e, ref.c2s()).astype(np.float64))) - (-10.685918926843847)) < 1e-9


# ---------------------------------------------------------------------------------------------------------------------
# Integrals out of the shipped kernels
NE = [[0, [1.0e5, 0.002], [3000., 0.02], [100., 0.2], [8.0, 0.5], [0.5, 0.4]],
      [1, [20.0, 0.3], [1.5, 0.6], [0.15, 0.3]],
      [2, [8.0, 0.10], [3.2, 0.30], [1.3, 0.40], [0.55, 0.30], [0.22, 0.10]],            # 5 primitives: 25 pairs
      [3, [20.0, 0.15], [6.0, 0.35], [2.0, 0.40], [0.7, 0.25], [0.25, 0.10]]]             # 5 primitives: 25 pairs
HE = [[0, [30., 0.2], [5., 0.5], [0.8, 0.5]],
      [2, [4.0, 0.5, 0.1], [1.1, 0.5, -0.6], [0.3, 0.2, 1.0]],                            # nctr = 2
      [3, [12.0, 1.0, 0.4], [1.5, 0.3, 1.0]]]                                              # nctr = 2
# one primitive per shell, exponents from 0.05 to 1e5; the atoms are 0.57 bohr (spdf) and 17.9 bohr (far) apart
O1 = [[0, [1.0e5, 1.0]], [1, [0.9, 1.0]], [2, [0.6, 1.0]], [3, [0.8, 1.0]]]
C1 = [[0, [0.05, 1.0]], [1, [40.0, 1.0]], [2, [3.0, 1.0]], [3, [0.3, 1.0]]]
FAR_A = [[0, [2.0, 1.0]], [1, [0.05, 1.0]], [2, [25.0, 1.0]], [3, [6.0, 1.0]]]
FAR_B = [[0, [500.0, 1.0]], [1, [3.0, 1.0]], [2, [0.1, 1.0]], [3, [1.5, 1.0]]]
SYSTEMS = {
    'contracted': dict(atom='Ne 0 0 0; He 1 2 2', basis={'Ne': NE, 'He': HE}),
    'spdf': dict(atom='O 0 0 0; C 0.25 -0.5 0.125', basis={'O': O1, 'C': C1}),
    'far': dict(atom='Cl 0 0 0; Ar 0 8 -16', basis={'Cl': FAR_A, 'Ar': FAR_B}),
}
OMEGAS = (0.0, 0.35, 8.0, -0.4)

def PAIR_ID(l1, l2):
    """pair class id l1 (l1 + 1) / 2 + l2, l1 >= l2 (scalars or arrays)"""
    hi, lo = np.maximum(l1, l2), np.minimum(l1, l2)
    return hi * (hi + 1) // 2 + lo


PAIR_LS = {PAIR_ID(a, b): (a, b) for a in range(4) for b in range(a + 1)}
# The labels below restate launch decisions of the library: use_swapped and choose_np (with B2_NVMAX) in
# pyscf_b200/csrc/jk_classes.cuh, TpqCfg::eligible in jk_tpq.cuh.  test_class_labels_match_kernel_sources reads those
# sources and fails when they no longer match.
SWAPPED = {(6, 4), (7, 4), (6, 2), (7, 5)}           # use_swapped: (hi, lo) pairs run with the smaller class as bra
NVMAX = 30                                           # B2_NVMAX
L_CHAR = 'spdf'


def _choose_np(ni, nj, nkl, nvmax=NVMAX):
    """choose_np of jk_classes.cuh."""
    eff = lambda g: (32 // g) * g * 1000 // 32 if g <= 32 else g * 1000 // (((g + 31) // 32) * 32)
    best, best_eff = 0, -1
    for np_ in range(1, nj + 1):
        if nj % np_ or ni * nj // np_ > nvmax:
            continue
        if best and ni * nj // np_ < 15:
            break
        if nkl * np_ > 512:
            break
        if eff(nkl * np_) > best_eff + 60:
            best, best_eff = np_, eff(nkl * np_)
    return best or nj


def launched(cb, ck):
    """(bra pair class, ket pair class) of the kernel that computes a quartet of pair classes cb, ck."""
    hi, lo = max(cb, ck), min(cb, ck)
    return (lo, hi) if (hi, lo) in SWAPPED else (hi, lo)


def family(cls):
    la, lb = PAIR_LS[cls[0]]
    lc, ld = PAIR_LS[cls[1]]
    nc = R.ncart
    tpq = nc(la) * nc(lb) * nc(lc) * nc(ld) <= 36 and (la + lb + lc + ld) // 2 + 1 <= 3 and \
        _choose_np(nc(la), nc(lb), nc(lc) * nc(ld)) == 1
    return 'tpq' if tpq else 'block'


def class_name(cls):
    (la, lb), (lc, ld) = PAIR_LS[cls[0]], PAIR_LS[cls[1]]
    return '(%s%s|%s%s)' % (L_CHAR[la], L_CHAR[lb], L_CHAR[lc], L_CHAR[ld])


ALL_CLASSES = sorted({launched(a, b) for a in range(10) for b in range(10)})
assert len(ALL_CLASSES) == 55


def test_class_labels_match_kernel_sources():
    """The swapped orientations, B2_NVMAX and the thread-per-quartet rule restated above are the library's."""
    import os
    import re
    src = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), 'pyscf_b200', 'csrc')
    cls = open(os.path.join(src, 'jk_classes.cuh')).read()
    body = re.search(r'constexpr bool use_swapped\(int hi, int lo\)\s*\{(.*?)\}', cls, re.S).group(1)
    pairs = {(int(a), int(b)) for a, b in re.findall(r'hi == (\d+) && lo == (\d+)', body)}
    assert pairs == SWAPPED, pairs
    assert int(re.search(r'#define B2_NVMAX (\d+)', cls).group(1)) == NVMAX
    tpq = open(os.path.join(src, 'jk_tpq.cuh')).read()
    assert 'eligible = (NOUT <= 36) && (C::NR <= 3) && (C::NP == 1);' in tpq
    assert 'return nout <= 36 && nr <= 3 && choose_np(ncart(la), ncart(lb), ncart(lc) * ncart(ld)) == 1;' in cls
    # DESIGN.md §4.1: 12 thread-per-quartet classes, 43 block classes (tpq_class of jk_classes.cuh over the 55 classes
    # as launched)
    assert sum(family(c) == 'tpq' for c in ALL_CLASSES) == 12


def sph_offsets(ref):
    return np.cumsum([0] + [2 * s.l + 1 for s in ref.segs])


def cart_offsets(ref):
    return np.cumsum([0] + [R.ncart(s.l) for s in ref.segs])


def block_max(t, off):
    for ax in range(4):
        t = np.maximum.reduceat(t, off[:-1], axis=ax)
    return t


def block_ratio(err, sblk, off):
    """Per shell-quartet block: max error / S (inf where S = 0 and the error is not exactly 0)."""
    e = block_max(err, off)
    with np.errstate(divide='ignore', invalid='ignore'):
        r = np.where(sblk > 0, e / np.where(sblk > 0, sblk, 1), np.where(e > 0, np.inf, 0.0))
    return r


_REF = {}


def reference(name, omega):
    """(Reference, eri_cart, S_cart, {n_roots: x values}) of a system, cached per operator."""
    key = (name, omega)
    if key not in _REF:
        mol = gto.M(unit='Bohr', **SYSTEMS[name])
        ref = R.Reference(mol._atm, mol._bas, mol._env)
        xlog = {}
        e, s = ref.eri_cart(omega, xlog)
        _REF[key] = (ref, e, s.astype(np.float64), {n: np.concatenate(v) for n, v in xlog.items()})
    return _REF[key]


def kernel_eri(opt, nao, route, shard=None):
    """Every (ij|kl) of the handle from unit densities.  K route: hermi = 0, D = E_jk, K_il = (ij|kl).  J route:
    D = E_kl + E_lk (E_kk on the diagonal), J_ij = 2 (ij|kl) (or (ij|kk))."""
    if shard is not None:
        opt.handle.check(opt.handle.lib.b200jk_set_shard(opt.handle._h, *shard), 'b200jk_set_shard')
    if route == 'K':
        dms = np.eye(nao * nao).reshape(nao * nao, nao, nao)
        _, vk = opt.get_jk(dms, hermi=0, with_j=False)
        return vk.reshape(nao, nao, nao, nao).transpose(2, 0, 1, 3)
    kk, ll = np.tril_indices(nao)
    d = np.zeros((len(kk), nao, nao))
    d[np.arange(len(kk)), kk, ll] = 1.0
    d[np.arange(len(kk)), ll, kk] = 1.0
    vj, _ = opt.get_jk(d, hermi=1, with_k=False)
    vj[kk != ll] *= 0.5
    eri = np.zeros((nao,) * 4)
    eri[:, :, kk, ll] = vj.transpose(1, 2, 0)
    eri[:, :, ll, kk] = vj.transpose(1, 2, 0)
    return eri


class Tally:
    """Largest error / S per launched class and route, and the coverage of the runs."""

    def __init__(self):
        self.worst = {}
        self.xs = {}
        self.lines = []

    def add(self, label, route, ref, eri_ref, s_ref, eri, cart, xlog, floor=0.0):
        T = None if cart else ref.c2s()
        off = cart_offsets(ref) if cart else sph_offsets(ref)
        if cart:
            er, sr = eri_ref.astype(np.float64), s_ref
        else:
            er = R.to_sph(eri_ref, T).astype(np.float64)
            sr = R.to_sph(s_ref.astype(R.LD), np.abs(T)).astype(np.float64)
        sb = block_max(sr, off)
        if route == 'K':
            sb = np.maximum(sb, sb.transpose(0, 2, 1, 3))
        if floor:
            sb = np.where(sb > 0, np.maximum(sb, floor * sb.max()), 0.0)
        ratio = block_ratio(np.abs(eri - er), sb, off) / EPS
        ls = np.array([s.l for s in ref.segs])
        pid = PAIR_ID(ls[:, None], ls[None, :])
        bad = []
        for cls in ALL_CLASSES:
            m = np.zeros_like(ratio, dtype=bool)
            for cb, ck in ((cls[0], cls[1]), (cls[1], cls[0])):
                m |= (pid[:, :, None, None] == cb) & (pid[None, None] == ck)
            if not m.any():
                continue
            r = ratio[m]
            key = (cls, route)
            self.worst[key] = max(self.worst.get(key, 0.0), float(r.max()))
            if r.max() > KAPPA:
                q = np.argwhere(m & (ratio == r.max()))[0]
                bad.append('%s %s [%s route, %s]: shell quartet %s, error/S = %.3g eps, bar %d eps (%.2e)' % (
                    class_name(cls), family(cls), route, label, tuple(int(v) for v in q), r.max(), KAPPA, BAR))
        for n, x in xlog.items():
            self.xs.setdefault(n, []).append(x)
        self.lines.append('%-32s %s route: worst %.1f eps' % (label, route, ratio[np.isfinite(ratio)].max()))
        assert not bad, '\n'.join(bad)

    def report(self, what):
        print('%s: largest error / S per class, in units of eps (K route, J route); bar %d eps' % (what, KAPPA))
        for cls in ALL_CLASSES:
            print('  %-8s %-5s %7.1f %7.1f' % (class_name(cls), family(cls), self.worst.get((cls, 'K'), -1),
                                                 self.worst.get((cls, 'J'), -1)))

    def check_coverage(self):
        for route in ('K', 'J'):
            missing = [class_name(c) for c in ALL_CLASSES if (c, route) not in self.worst]
            assert not missing, 'classes never reached in the %s route: %s' % (route, missing)
        assert {family(c) for c in ALL_CLASSES} == {'tpq', 'block'}
        for (hi, lo) in SWAPPED:
            assert ((lo, hi), 'K') in self.worst and ((lo, hi), 'J') in self.worst
        counts = {}
        for n in range(1, 8):
            x = np.concatenate(self.xs.get(n, [np.zeros(0)]))
            counts[n] = (int((x == 0).sum()), int(((x > 0) & (x < 100)).sum()), int((x >= 100).sum()))
            assert all(c > 0 for c in counts[n]), 'n=%d: primitive quartets at x = 0, 0 < x < 100, x >= 100: %s' % (n, counts[n])
        print('primitive quartets per root count n (x = 0, 0 < x < 100, x >= 100):', counts)


def check_contracted_coverage():
    """The contracted system carries d and f pairs beyond MAX_PRIM_PER_PAIR = 16, nctr = 2 d and f shells, and pair classes
    whose kets have different primitive counts after the split."""
    ref = reference('contracted', 0.0)[0]
    mol = gto.M(unit='Bohr', **SYSTEMS['contracted'])
    assert {2, 3} <= {int(b[1]) for b in mol._bas if b[3] > 1}
    big = [(p.la, p.lb) for p in ref.pairs.values() if p.nprim > 16]
    assert any(l >= 2 for ab in big for l in ab) and (2, 2) in big and (3, 3) in big
    per_class = {}
    for p in ref.pairs.values():
        cnt = [min(16, p.nprim - p0) for p0 in range(0, p.nprim, 16)]
        per_class.setdefault(PAIR_ID(p.la, p.lb), set()).update(cnt)
    assert all(len(per_class[PAIR_ID(a, b)]) > 1 for a, b in ((2, 2), (3, 2), (3, 3)))


def run_case(tally, lib, name, omega, cart=False, routes=('K', 'J')):
    ref, e, s, xlog = reference(name, omega)
    mol = gto.M(unit='Bohr', cart=cart, **SYSTEMS[name])
    nao = ref.ncart if cart else int(sph_offsets(ref)[-1])
    opt = VHFOpt(mol, direct_scf_tol=0.0, omega=omega, libpath=lib)
    label = '%s%s omega=%g' % (name, ' cart' if cart else '', omega)
    for route in routes:
        t = time.time()
        eri = kernel_eri(opt, nao, route)
        tally.add(label, route, ref, e, s, eri, cart, xlog if route == 'K' else {}, FLOOR.get(name, 0.0))
        tally.lines[-1] += ' (%.0f s)' % (time.time() - t)
        print(tally.lines[-1], flush=True)
    opt.close()


def single_density_j(lib, name, omega, pairs):
    """The n_dm = 1 J path (the register-resident J[ij] flush of the block kernels) on a few unit densities."""
    ref, e, s, _ = reference(name, omega)
    mol = gto.M(unit='Bohr', **SYSTEMS[name])
    off = sph_offsets(ref)
    T = ref.c2s()
    er = R.to_sph(e, T).astype(np.float64)
    sb = block_max(R.to_sph(s.astype(R.LD), np.abs(T)).astype(np.float64), off)
    seg = np.searchsorted(off, np.arange(off[-1]), side='right') - 1
    opt = VHFOpt(mol, direct_scf_tol=0.0, omega=omega, libpath=lib)
    for k, l in pairs:
        d = np.zeros((off[-1], off[-1]))
        d[k, l] = d[l, k] = 1.0
        vj, _ = opt.get_jk(d, hermi=1, with_k=False)
        got = vj / (1.0 if k == l else 2.0)
        scale = sb[:, :, seg[k], seg[l]][seg][:, seg]
        r = np.abs(got - er[:, :, k, l]) / np.where(scale > 0, scale, 1) / EPS
        assert np.all(np.where(scale > 0, r <= KAPPA, got == er[:, :, k, l])), ('n_dm = 1 J', name, omega, k, l, r.max())
    opt.close()


def test_eri_classes_emulated(emu_lib):
    """Every class, both routes, on the CPU emulation: spdf (single primitives, all four operators, and omega = 8 in
    Cartesian AOs) and the contracted system (Coulomb)."""
    tally = Tally()
    for omega in OMEGAS:
        run_case(tally, emu_lib, 'spdf', omega)
    run_case(tally, emu_lib, 'spdf', 8.0, cart=True)
    run_case(tally, emu_lib, 'contracted', 0.0)
    tally.report('CPU emulation')
    tally.check_coverage()
    check_contracted_coverage()
    single_density_j(emu_lib, 'contracted', 0.0, [(0, 0), (30, 12), (40, 25), (20, 9)])


def test_eri_experimental_layouts_emulated(emu_lib_experimental):
    """The experimental lane layouts (B2_PBMAX=4, B2_PPW=1, B2_TPQ_KOUTER=1) on the same integrals.  `contracted` gives
    the primitive batches of the block kernels several primitive quartets of d and f pairs (up to 16 x 16 per quartet,
    batches that cross bra primitives); spdf, with one primitive quartet per shell quartet, only ever runs tail batches.
    (ff| bra classes keep one quartet per round in every build, jk_classes.cuh.)"""
    tally = Tally()
    for omega in (0.0, -0.4):
        run_case(tally, emu_lib_experimental, 'spdf', omega)
    run_case(tally, emu_lib_experimental, 'contracted', 0.0)
    tally.report('CPU emulation, experimental layouts')


def check_shard(lib, name, omega):
    """Two ranks of b200jk_set_shard: the partial K of every unit density sums to the unsharded result."""
    ref, e, s, _ = reference(name, omega)
    mol = gto.M(unit='Bohr', **SYSTEMS[name])
    nao = int(sph_offsets(ref)[-1])
    opt = VHFOpt(mol, direct_scf_tol=0.0, omega=omega, libpath=lib)
    full = kernel_eri(opt, nao, 'K')
    part = [kernel_eri(opt, nao, 'K', shard=(r, 2)) for r in range(2)]
    opt.close()
    assert np.abs(part[0]).max() > 0 and np.abs(part[1]).max() > 0
    assert np.abs(part[0] + part[1] - full).max() <= 64 * EPS * np.abs(full).max()
    tally = Tally()
    tally.add('%s omega=%g shards 0+1' % (name, omega), 'K', ref, e, s, part[0] + part[1], False, {})


def test_eri_shard_split_emulated(emu_lib):
    check_shard(emu_lib, 'spdf', 0.0)


DEVICE_CASES = {
    'spdf': [(o, False) for o in OMEGAS],
    'far': [(o, False) for o in OMEGAS],
    'contracted': [(0.0, False), (-0.4, False)],
    'contracted_cart': [(0.35, True)],
}


@pytest.mark.gpu
@pytest.mark.parametrize('case', list(DEVICE_CASES))
def test_eri_classes_device(case):
    """Every system on the H100, both routes: spdf and far with all four operators, the contracted system with the
    Coulomb and erfc operators in spherical AOs (plus the n_dm = 1 J path and the coverage checks: it alone reaches all
    55 classes and x on both sides of 100 for n = 1..7) and with omega = 0.35 in Cartesian AOs."""
    name = case.split('_')[0]
    tally = Tally()
    for omega, cart in DEVICE_CASES[case]:
        run_case(tally, None, name, omega, cart=cart)
    tally.report('H100, %s' % case)
    if case == 'contracted':
        tally.check_coverage()
        check_contracted_coverage()
        single_density_j(None, name, 0.0, [(0, 0), (30, 12), (40, 25), (20, 9)])
        single_density_j(None, name, -0.4, [(30, 12), (40, 25)])


@pytest.mark.gpu
def test_eri_shard_split_device():
    check_shard(None, 'spdf', -0.4)
