"""High-precision two-electron integrals for the tests: plain McMurchie-Davidson in np.longdouble.

Input: libcint-layout tables (_atm, _bas, _env).  Output: contracted Cartesian (ij|kl) blocks, the bare monomials
x^lx y^ly z^lz exp(-a r^2) times the _env coefficients and libcint's s/p factors (the functions of int2e_cart), and for
every element S_abs, the same sum with every primitive-quartet contribution and every contraction coefficient taken in
absolute value (the scale of the accuracy bars).  `c2s_matrix` gives the real-solid-harmonic transforms, so spherical
results can be compared too.

Operators: omega = 0 Coulomb; omega > 0 erf(omega r)/r, i.e. alpha -> alpha w^2/(w^2+alpha) and the prefactor times
sqrt(w^2/(w^2+alpha)); omega < 0 erfc(|omega| r)/r = Coulomb - erf.

General contractions are split into one segment per contraction column, dropping zero coefficients, and primitive pairs
with |c_a c_b exp(-ab/(a+b) |AB|^2)| < prim_cut are dropped; both are what the library does with its device shells
(b200jk_create2), so a comparison measures the arithmetic and not the cut.

Per primitive quartet: (ab|cd) = 2 pi^(5/2) / (p q sqrt(p+q)) sum_{h,h'} E^ab_h (-1)^|h'| R_{h+h'} E^cd_h', vectorised as
E_bra . R . E_ket^T over the Hermite indices h = (t,u,v), t+u+v <= la+lb, and over all primitive quartets of a shell quartet.
"""
import numpy as np

LD = np.longdouble
PI = np.arccos(LD(-1))
LONGDOUBLE_OK = np.finfo(np.longdouble).eps <= 1e-18
SKIP_REASON = 'np.longdouble has eps %.1e here: the reference needs 80-bit or wider long double' % np.finfo(np.longdouble).eps

ATM_SLOTS, BAS_SLOTS = 6, 8
PRIM_CUT = 1e-18          # the library's cut on |c_a c_b K_ab| of a primitive pair (host_common.hpp)
_SP_FAC = {0: LD(1) / (2 * np.sqrt(PI)), 1: np.sqrt(LD(3) / (4 * PI))}


def cart_comps(l):
    """libcint Cartesian order: lx descending, then ly descending."""
    return [(x, y, l - x - y) for x in range(l, -1, -1) for y in range(l - x, -1, -1)]


def ncart(l):
    return (l + 1) * (l + 2) // 2


def _herm(L):
    return [(t, u, v) for t in range(L + 1) for u in range(L + 1 - t) for v in range(L + 1 - t - u)]


# ---------------------------------------------------------------------------------------------------------------------
def boys(mmax, x):
    """F_m(x) for m = 0..mmax in long double: [mmax+1, *x.shape].

    x < 50: the series F_M(x) = e^-x sum_k (2x)^k / ((2M+1)(2M+3)...(2M+2k+1)) for the top order, then the stable downward
    recursion F_m = (2x F_{m+1} + e^-x) / (2m+1).  x >= 50: F_0 = sqrt(pi/x)/2 (erfc(sqrt x) < 2e-23 is below the long
    double epsilon) and the upward recursion F_{m+1} = ((2m+1) F_m - e^-x) / (2x), stable for x > m + 1/2."""
    x = np.asarray(x, dtype=LD)
    shape = x.shape
    x = x.reshape(-1)
    F = np.empty((mmax + 1, x.size), dtype=LD)
    ex = np.exp(-x)
    lo = x < 50
    if lo.any():
        xs, es = x[lo], ex[lo]
        term = np.full(xs.shape, LD(1) / (2 * mmax + 1))
        s = term.copy()
        k = 0
        while True:
            k += 1
            term = term * (2 * xs) / (2 * mmax + 2 * k + 1)
            s += term
            if not np.any(term > s * LD(1e-22)):
                break
        Fl = np.empty((mmax + 1, xs.size), dtype=LD)
        Fl[mmax] = es * s
        for m in range(mmax - 1, -1, -1):
            Fl[m] = (2 * xs * Fl[m + 1] + es) / (2 * m + 1)
        F[:, lo] = Fl
    hi = ~lo
    if hi.any():
        xs, es = x[hi], ex[hi]
        Fh = np.empty((mmax + 1, xs.size), dtype=LD)
        Fh[0] = np.sqrt(PI / xs) / 2
        for m in range(mmax):
            Fh[m + 1] = ((2 * m + 1) * Fh[m] - es) / (2 * xs)
        F[:, hi] = Fh
    return F.reshape((mmax + 1,) + shape)


# ---------------------------------------------------------------------------------------------------------------------
def _hermite_1d(li, lj, PA, PB, p):
    """E[i][j][t] arrays over primitive pairs (1-D Hermite expansion of x_A^i x_B^j, without the Gaussian factor)."""
    n = PA.shape[0]
    E = np.zeros((li + 1, lj + 1, li + lj + 2, n), dtype=LD)
    E[0, 0, 0] = 1
    h = 1 / (2 * p)
    for i in range(li + 1):
        for j in range(lj + 1):
            if i == 0 and j == 0:
                continue
            if i > 0:
                src, X, a, b = E[i - 1, j], PA, i - 1, j
            else:
                src, X, a, b = E[i, j - 1], PB, i, j - 1
            for t in range(a + b + 2):
                v = X * src[t]
                if t > 0:
                    v = v + h * src[t - 1]
                if t + 1 <= a + b:
                    v = v + (t + 1) * src[t + 1]
                E[i, j, t] = v
    return E


class _Seg:
    def __init__(self, l, r, e, c, ao_cart):
        self.l, self.r, self.e, self.c, self.ao_cart = l, r, e, c, ao_cart


def segments(atm, bas, env):
    """One segment per (shell, contraction column), with its nonzero primitives; Cartesian AO offsets in _bas order."""
    atm = np.asarray(atm).reshape(-1, ATM_SLOTS)
    bas = np.asarray(bas).reshape(-1, BAS_SLOTS)
    env = np.asarray(env, dtype=np.float64)
    segs, off = [], 0
    for b in bas:
        l, npr, nc = int(b[1]), int(b[2]), int(b[3])
        r = env[atm[b[0], 1]:atm[b[0], 1] + 3].astype(LD)
        e = env[b[5]:b[5] + npr]
        cm = env[b[6]:b[6] + npr * nc].reshape(nc, npr)
        for c in range(nc):
            keep = cm[c] != 0.0
            segs.append(_Seg(l, r, e[keep].copy(), cm[c][keep].copy(), off))
            off += ncart(l)
    return segs, off


class _Pair:
    """Surviving primitive pairs of two segments and their Hermite expansions E[npp, na*nb, nherm], the coefficients,
    libcint's s/p factors and exp(-ab/p |AB|^2) folded in."""

    def __init__(self, A, B, prim_cut):
        self.A, self.B = A, B
        self.la, self.lb = A.l, B.l
        AB = A.r - B.r
        r2 = float(np.dot(AB.astype(np.float64), AB.astype(np.float64)))
        ia, ib = np.meshgrid(np.arange(len(A.e)), np.arange(len(B.e)), indexing='ij')
        ia, ib = ia.ravel(), ib.ravel()
        ea, eb = A.e[ia], B.e[ib]
        # the library's cut, in double precision as the library evaluates it
        cc64 = A.c[ia] * B.c[ib] * np.exp(-ea * eb / (ea + eb) * r2)
        keep = np.abs(cc64) >= prim_cut
        ia, ib = ia[keep], ib[keep]
        self.nprim = len(ia)
        ea, eb = A.e[ia].astype(LD), B.e[ib].astype(LD)
        p = ea + eb
        P = (ea[:, None] * A.r[None] + eb[:, None] * B.r[None]) / p[:, None]
        K = np.exp(-ea * eb / p * np.dot(AB, AB))
        coef = A.c[ia].astype(LD) * B.c[ib].astype(LD) * K * _SP_FAC.get(A.l, LD(1)) * _SP_FAC.get(B.l, LD(1))
        self.p, self.P = p, P
        L = A.l + B.l
        self.herm = _herm(L)
        Ed = [_hermite_1d(A.l, B.l, P[:, d] - A.r[d], P[:, d] - B.r[d], p) for d in range(3)]
        ca, cb = cart_comps(A.l), cart_comps(B.l)
        E = np.zeros((self.nprim, len(ca) * len(cb), len(self.herm)), dtype=LD)
        for a, (ax, ay, az) in enumerate(ca):
            for b, (bx, by, bz) in enumerate(cb):
                for h, (t, u, v) in enumerate(self.herm):
                    if t <= ax + bx and u <= ay + by and v <= az + bz:
                        E[:, a * len(cb) + b, h] = Ed[0][ax, bx, t] * Ed[1][ay, by, u] * Ed[2][az, bz, v] * coef
        self.E = E


def _rtensor(L, alpha, PQ, F):
    """R^0_{tuv} for t+u+v <= L over primitive quartets: dict (t,u,v) -> array.  F: Boys values [L+1, nq]."""
    prev = {}
    for n in range(L, -1, -1):
        cur = {(0, 0, 0): (-2 * alpha) ** n * F[n]}
        for (t, u, v) in _herm(L - n):
            if t + u + v == 0:
                continue
            if t > 0:
                val = PQ[:, 0] * prev[(t - 1, u, v)]
                if t > 1:
                    val = val + (t - 1) * prev[(t - 2, u, v)]
            elif u > 0:
                val = PQ[:, 1] * prev[(t, u - 1, v)]
                if u > 1:
                    val = val + (u - 1) * prev[(t, u - 2, v)]
            else:
                val = PQ[:, 2] * prev[(t, u, v - 1)]
                if v > 1:
                    val = val + (v - 1) * prev[(t, u, v - 2)]
            cur[(t, u, v)] = val
        prev = cur
    return prev


_GATHER = {}


def _gather(Lb, Lk):
    """Index of R_{h+h'} in the list _herm(Lb+Lk) and the sign (-1)^|h'|, for every (h, h') of _herm(Lb) x _herm(Lk)."""
    if (Lb, Lk) not in _GATHER:
        pos = {h: i for i, h in enumerate(_herm(Lb + Lk))}
        hb, hk = _herm(Lb), _herm(Lk)
        idx = np.array([[pos[(t + t2, u + u2, v + v2)] for (t2, u2, v2) in hk] for (t, u, v) in hb], dtype=np.int64)
        sign = np.array([[-1.0 if sum(h2) & 1 else 1.0 for h2 in hk] for _ in hb]).astype(LD)
        _GATHER[Lb, Lk] = (idx, sign)
    return _GATHER[Lb, Lk]


def _quartet_one_op(bra, ket, omega):
    """Per-primitive-quartet contributions V[nb, nk, nab, ncd] for one operator (omega >= 0), and the x of every quartet."""
    p, q = bra.p[:, None], ket.p[None, :]
    PQ = (bra.P[:, None, :] - ket.P[None, :, :]).reshape(-1, 3)
    alpha = (p * q / (p + q)).reshape(-1)
    pref = (2 * PI ** LD(2.5) / (p * q * np.sqrt(p + q))).reshape(-1)
    if omega > 0:
        w2 = LD(omega) ** 2
        theta = w2 / (w2 + alpha)
        alpha = alpha * theta
        pref = pref * np.sqrt(theta)
    L = bra.la + bra.lb + ket.la + ket.lb
    x = alpha * (PQ ** 2).sum(axis=1)
    R = _rtensor(L, alpha, PQ, boys(L, x))
    nb, nk = bra.nprim, ket.nprim
    idx, sign = _gather(bra.la + bra.lb, ket.la + ket.lb)
    Rarr = np.stack([R[h] for h in _herm(L)]) * pref                           # [nherm(L), nq]
    M = Rarr[idx] * sign[:, :, None]                                           # [hb, hk, nq]
    nhb, nhk = len(bra.herm), len(ket.herm)
    nab, ncd = bra.E.shape[1], ket.E.shape[1]
    M = M.reshape(nhb, nhk, nb, nk).transpose(2, 0, 3, 1)                     # [nb, hb, nk, hk]
    # value, long double: T[b] = sum_{k,h'} M[b,:,k,h'] E_k[k,:,h'],  V = sum_{b,h} E_b[b,:,h] T[b,h,:]
    T = np.matmul(M.reshape(nb, nhb, nk * nhk), ket.E.transpose(0, 2, 1).reshape(nk * nhk, ncd))    # [nb, hb, ncd]
    val = np.matmul(bra.E.transpose(1, 0, 2).reshape(nab, nb * nhb), T.reshape(nb * nhb, ncd))
    # S_abs, a scale only: double precision is enough for the per-quartet absolute values
    M64 = M.astype(np.float64).transpose(0, 2, 1, 3)                           # [nb, nk, hb, hk]
    V64 = np.matmul(bra.E.astype(np.float64)[:, None], np.matmul(M64, ket.E.astype(np.float64).transpose(0, 2, 1)[None]))
    return val, np.abs(V64).sum(axis=(0, 1)), x


def quartet(bra, ket, omega=0.0):
    """Contracted Cartesian block [nab, ncd] of (bra|ket), its S_abs, and the x values the quadrature sees."""
    if bra.nprim == 0 or ket.nprim == 0:
        z = np.zeros((bra.E.shape[1], ket.E.shape[1]), dtype=LD)
        return z, z.copy(), np.zeros(0)
    if omega >= 0:
        return _quartet_one_op(bra, ket, omega)
    vc, sc, xc = _quartet_one_op(bra, ket, 0.0)
    ve, se, xe = _quartet_one_op(bra, ket, -omega)
    return vc - ve, sc + se, np.concatenate([xc, xe])


class Reference:
    """All contracted Cartesian integrals of a basis, computed once per operator."""

    def __init__(self, atm, bas, env, prim_cut=PRIM_CUT):
        self.segs, self.ncart = segments(atm, bas, env)
        self.pairs = {}
        for i, A in enumerate(self.segs):
            for j, B in enumerate(self.segs[:i + 1]):
                self.pairs[i, j] = _Pair(A, B, prim_cut)

    def eri_cart(self, omega=0.0, xlog=None):
        """(eri[n,n,n,n], S_abs[n,n,n,n]) in long double, Cartesian AOs in _bas order.  xlog: optional dict n_roots -> list
        of arrays of the x values the quadrature of each shell quartet sees."""
        n = self.ncart
        eri = np.zeros((n,) * 4, dtype=LD)
        sab = np.zeros((n,) * 4, dtype=LD)
        keys = sorted(self.pairs)
        for ib, kb in enumerate(keys):
            for kk in keys[:ib + 1]:
                bra, ket = self.pairs[kb], self.pairs[kk]
                v, s, x = quartet(bra, ket, omega)
                if xlog is not None and len(x):
                    xlog.setdefault((bra.la + bra.lb + ket.la + ket.lb) // 2 + 1, []).append(x.astype(np.float64))
                A, B, C, D = bra.A, bra.B, ket.A, ket.B
                na, nb, nc, nd = ncart(A.l), ncart(B.l), ncart(C.l), ncart(D.l)
                v = v.reshape(na, nb, nc, nd)
                s = s.reshape(na, nb, nc, nd)
                sa, sb, sc, sd = (slice(X.ao_cart, X.ao_cart + ncart(X.l)) for X in (A, B, C, D))
                for blk, src in ((eri, v), (sab, s)):
                    blk[sa, sb, sc, sd] = src
                    blk[sb, sa, sc, sd] = src.transpose(1, 0, 2, 3)
                    blk[sa, sb, sd, sc] = src.transpose(0, 1, 3, 2)
                    blk[sb, sa, sd, sc] = src.transpose(1, 0, 3, 2)
                    blk[sc, sd, sa, sb] = src.transpose(2, 3, 0, 1)
                    blk[sd, sc, sa, sb] = src.transpose(3, 2, 0, 1)
                    blk[sc, sd, sb, sa] = src.transpose(2, 3, 1, 0)
                    blk[sd, sc, sb, sa] = src.transpose(3, 2, 1, 0)
        return eri, sab

    def c2s(self):
        """Block-diagonal Cartesian -> spherical AO map T[nsph, ncart] (real solid harmonics, libcint's order and
        normalisation): eri_sph = T (x) T (x) T (x) T applied to eri_cart."""
        blocks = [c2s_matrix(s.l) for s in self.segs]
        ns = sum(b.shape[0] for b in blocks)
        T = np.zeros((ns, self.ncart), dtype=LD)
        r = 0
        for s, b in zip(self.segs, blocks):
            T[r:r + b.shape[0], s.ao_cart:s.ao_cart + b.shape[1]] = b
            r += b.shape[0]
        return T


def c2s_matrix(l):
    """[2l+1, ncart(l)] real-solid-harmonic coefficients of the Cartesian monomials, rows m = -l..l (p: x, y, z), times
    sqrt((2l+1)/(4 pi)) (Helgaker, Jorgensen, Olsen eq. 6.4.47); for l <= 1 the identity, as libcint's s/p factors are
    already in the Cartesian functions."""
    from math import comb, factorial
    nc = ncart(l)
    if l <= 1:
        return np.eye(nc, dtype=LD)
    comps = cart_comps(l)
    T = np.zeros((2 * l + 1, nc), dtype=LD)
    ang = np.sqrt(LD(2 * l + 1) / (4 * PI))
    for m in range(-l, l + 1):
        am = abs(m)
        N = np.sqrt(LD(2 * factorial(l + am) * factorial(l - am)) / (2 if m == 0 else 1)) / LD(2 ** am * factorial(l))
        vm2 = 1 if m < 0 else 0            # 2 v_m
        for t in range((l - am) // 2 + 1):
            for u in range(t + 1):
                for v2 in range(vm2, 2 * ((am - vm2) // 2) + vm2 + 1, 2):
                    sgn = -1 if (t + (v2 - vm2) // 2) & 1 else 1
                    C = sgn * LD(comb(l, t) * comb(l - t, am + t) * comb(t, u) * comb(am, v2)) / LD(4) ** t
                    lx, ly, lz = 2 * t + am - 2 * u - v2, 2 * u + v2, l - 2 * t - am
                    if min(lx, ly, lz) < 0:
                        continue
                    T[m + l, comps.index((lx, ly, lz))] += ang * N * C
    return T


def to_sph(t4, T):
    """Apply the AO map T[ns, nc] to every index of a 4-index tensor."""
    for _ in range(4):
        t4 = np.tensordot(t4, T, axes=([0], [1]))     # cycles the axes: after four steps the order is restored
    return t4
