"""High-precision 3-center (ab|P) and 2-center (P|Q) integrals for the tests, on the 4-center machinery of eri_ref.py.

The fourth function is the unit function: an s "shell" of exponent 0 centred on the auxiliary function, without libcint's
s factor, so (ab|P) = (ab|P 1) and (P|Q) = (P 1|Q 1).  The pair (P, 1) has p = e_P, K = 1 and its product centre exactly on
P; its Hermite expansion is that of P alone.  The AO pairs keep the library's primitive cut; the auxiliary side has none
(the library drops only exact-zero coefficients there, as eri_ref.segments does).
"""
import numpy as np

from eri_ref import LD, PRIM_CUT, _SP_FAC, _Pair, _herm, _hermite_1d, c2s_matrix, cart_comps, ncart, quartet, segments


class UnitPair:
    """(segment A, unit function) as a ket or bra of eri_ref.quartet: the attributes of eri_ref._Pair."""

    def __init__(self, A):
        self.A, self.B = A, None
        self.la, self.lb = A.l, 0
        self.nprim = len(A.e)
        p = A.e.astype(LD)
        self.p, self.P = p, np.tile(A.r, (self.nprim, 1))
        self.herm = _herm(A.l)
        zero = np.zeros(self.nprim, dtype=LD)
        Ed = _hermite_1d(A.l, 0, zero, zero, p)
        coef = A.c.astype(LD) * _SP_FAC.get(A.l, LD(1))
        ca = cart_comps(A.l)
        E = np.zeros((self.nprim, len(ca), len(self.herm)), dtype=LD)
        for a, (ax, ay, az) in enumerate(ca):
            for h, (t, u, v) in enumerate(self.herm):
                if t <= ax and u <= ay and v <= az:
                    E[:, a, h] = Ed[ax, 0, t] * Ed[ay, 0, u] * Ed[az, 0, v] * coef
        self.E = E


def c2s_map(segs, n_cart):
    """Block-diagonal Cartesian -> spherical map T[nsph, n_cart] of a list of segments."""
    blocks = [c2s_matrix(s.l) for s in segs]
    T = np.zeros((sum(b.shape[0] for b in blocks), n_cart), dtype=LD)
    r = 0
    for s, b in zip(segs, blocks):
        T[r:r + b.shape[0], s.ao_cart:s.ao_cart + b.shape[1]] = b
        r += b.shape[0]
    return T


class DFReference:
    """3-center and 2-center integrals of an AO basis and an auxiliary basis (libcint tables each)."""

    def __init__(self, atm, bas, env, aux_atm, aux_bas, aux_env, prim_cut=PRIM_CUT):
        self.segs, self.ncart = segments(atm, bas, env)
        self.aux, self.naux_cart = segments(aux_atm, aux_bas, aux_env)
        self.pairs = {}
        for i, A in enumerate(self.segs):
            for j, B in enumerate(self.segs[:i + 1]):
                self.pairs[i, j] = _Pair(A, B, prim_cut)
        self.kets = [UnitPair(P) for P in self.aux]

    def int3c_cart(self, omega=0.0, xlog=None):
        """(v[n, n, naux], S_abs[n, n, naux]) in long double over Cartesian AOs and Cartesian auxiliary functions (the
        functions of int3c2e_cart).  xlog: optional dict n_roots -> list of arrays of the x values of each block."""
        n, m = self.ncart, self.naux_cart
        v = np.zeros((n, n, m), dtype=LD)
        s = np.zeros((n, n, m), dtype=LD)
        for bra in self.pairs.values():
            A, B = bra.A, bra.B
            sa, sb = slice(A.ao_cart, A.ao_cart + ncart(A.l)), slice(B.ao_cart, B.ao_cart + ncart(B.l))
            for C, ket in zip(self.aux, self.kets):
                val, sab, x = quartet(bra, ket, omega)
                if xlog is not None and len(x):
                    xlog.setdefault((A.l + B.l + C.l) // 2 + 1, []).append(x.astype(np.float64))
                sc = slice(C.ao_cart, C.ao_cart + ncart(C.l))
                for blk, src in ((v, val), (s, sab)):
                    src = src.reshape(ncart(A.l), ncart(B.l), ncart(C.l))
                    blk[sa, sb, sc] = src
                    blk[sb, sa, sc] = src.transpose(1, 0, 2)
        return v, s

    def int2c_cart(self, omega=0.0, xlog=None):
        """(v[naux, naux], S_abs[naux, naux]) in long double over Cartesian auxiliary functions (int2c2e_cart)."""
        m = self.naux_cart
        v = np.zeros((m, m), dtype=LD)
        s = np.zeros((m, m), dtype=LD)
        for i, (P, bra) in enumerate(zip(self.aux, self.kets)):
            for Q, ket in zip(self.aux[:i + 1], self.kets[:i + 1]):
                val, sab, x = quartet(bra, ket, omega)
                if xlog is not None and len(x):
                    xlog.setdefault((P.l + Q.l) // 2 + 1, []).append(x.astype(np.float64))
                sp, sq = slice(P.ao_cart, P.ao_cart + ncart(P.l)), slice(Q.ao_cart, Q.ao_cart + ncart(Q.l))
                for blk, src in ((v, val), (s, sab)):
                    blk[sp, sq] = src
                    blk[sq, sp] = src.T
        return v, s

    def c2s_ao(self):
        return c2s_map(self.segs, self.ncart)

    def c2s_aux(self):
        return c2s_map(self.aux, self.naux_cart)


def to_sph3(t3, Tao, Taux):
    """Apply the AO map to the first two indices and the auxiliary map to the third index of t3[n, n, naux]."""
    t3 = np.tensordot(Tao, t3, axes=([1], [0]))
    t3 = np.tensordot(Tao, t3, axes=([1], [1])).transpose(1, 0, 2)
    return np.tensordot(t3, Taux, axes=([2], [1]))


def to_sph2(t2, Taux):
    return Taux.dot(t2).dot(Taux.T)
