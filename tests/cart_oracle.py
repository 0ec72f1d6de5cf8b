"""Cartesian (mol.cart = True) counterparts of the oracle's density-fitting and one-electron helpers — TEST INFRASTRUCTURE ONLY.

The oracle library (oracle/liboracle.so) exports libcint-signature integral functions for both AO conventions; its fill
helpers and its one-electron matrix use the spherical ones.  This module calls int3c2e_cart / int2c2e_cart / int2e_cart shell
block by shell block instead, with the reference's conventions (pyscf/df/incore.py:129-220 for the tensor, pyscf/gto/mole.py
for the Cartesian functions: bare monomials with libcint's s and p factors).  The one-electron matrices are not in the oracle
library: overlap and kinetic energy come from exact Gauss-Hermite quadrature of the Cartesian Gaussian products, the nuclear
attraction from int3c2e_cart against a point-like s "auxiliary" function on each nucleus.  Pinned by tests/test_df_cart.py
against the spherical oracle (through the cart -> sph transform) and the reference's published energies.
"""
import ctypes
import os
from concurrent.futures import ThreadPoolExecutor

import numpy as np
import scipy.linalg

from oracle import oracle as O

_FAC = {0: 0.282094791773878143, 1: 0.488602511902919921}   # libcint's angular factors of s and p (make_c2c)
_NTHREAD = max(1, min(8, os.cpu_count() or 1))             # ctypes releases the GIL during the integral calls


def _fn(name):
    f = getattr(O.lib(), name)
    f.restype = ctypes.c_int
    return f


def _call(fn, shape, shls, atm, bas, env):
    out = np.zeros(int(np.prod(shape)))
    s = np.ascontiguousarray(shls, dtype=np.int32)
    fn(O._p(out), None, O._ip(s), O._ip(atm), ctypes.c_int(len(atm)), O._ip(bas), ctypes.c_int(len(bas)), O._p(env), None, None)
    return out.reshape(shape[::-1]).T          # Fortran-ordered block [d0, d1, ...]


def _pmap(f, items):
    with ThreadPoolExecutor(_NTHREAD) as ex:
        return list(ex.map(f, items))


def int3c2e_pairs(mol, auxmol, pairs):
    """(ij|P) over Cartesian functions for AO shell pairs [(ish, jsh), ...]: (out[naux, ncol], col0[npair]), pair p owning
    columns col0[p] + a*dj + b, as oracle.int3c2e_pairs.  Operator from mol._env[8]."""
    atm, bas, env = O.conc_mol(mol, auxmol)
    env[8] = mol._env[8]
    loc, aloc = mol.ao_loc_nr(cart=True), auxmol.ao_loc_nr(cart=True)
    pairs = np.asarray(pairs, dtype=np.int64).reshape(-1, 2)
    dims = (loc[pairs[:, 0] + 1] - loc[pairs[:, 0]]) * (loc[pairs[:, 1] + 1] - loc[pairs[:, 1]])
    col0 = np.concatenate([[0], np.cumsum(dims)[:-1]]).astype(np.int64)
    naux = int(aloc[-1])
    out = np.zeros((naux, int(dims.sum())))
    fn = _fn('int3c2e_cart')

    def one(p):
        i, j = pairs[p]
        di, dj = loc[i + 1] - loc[i], loc[j + 1] - loc[j]
        for k in range(auxmol.nbas):
            dk = aloc[k + 1] - aloc[k]
            b = _call(fn, (di, dj, dk), (i, j, mol.nbas + k), atm, bas, env)
            out[aloc[k]:aloc[k + 1], col0[p]:col0[p] + di * dj] = b.reshape(di * dj, dk).T
    _pmap(one, range(len(pairs)))
    return out, col0


def int3c2e(mol, auxmol):
    """(ij|P) over Cartesian functions, [nao, nao, naux] (aosym s1)."""
    loc = mol.ao_loc_nr(cart=True)
    nao = int(loc[-1])
    pairs = [(i, j) for i in range(mol.nbas) for j in range(i + 1)]
    blk, col0 = int3c2e_pairs(mol, auxmol, pairs)
    out = np.zeros((nao, nao, blk.shape[0]))
    for p, (i, j) in enumerate(pairs):
        di, dj = loc[i + 1] - loc[i], loc[j + 1] - loc[j]
        b = blk[:, col0[p]:col0[p] + di * dj].reshape(-1, di, dj).transpose(1, 2, 0)
        out[loc[i]:loc[i + 1], loc[j]:loc[j + 1]] = b
        out[loc[j]:loc[j + 1], loc[i]:loc[i + 1]] = b.transpose(1, 0, 2)
    return out


def int2c2e(auxmol, omega=None):
    """(P|Q) over Cartesian functions."""
    atm, bas, env = O._tables(auxmol)
    env = env.copy()
    if omega is not None:
        env[8] = omega
    loc = auxmol.ao_loc_nr(cart=True)
    n = int(loc[-1])
    out = np.zeros((n, n))
    fn = _fn('int2c2e_cart')

    def one(i):
        for j in range(i + 1):
            b = _call(fn, (loc[i + 1] - loc[i], loc[j + 1] - loc[j]), (i, j), atm, bas, env)
            out[loc[i]:loc[i + 1], loc[j]:loc[j + 1]] = b
            out[loc[j]:loc[j + 1], loc[i]:loc[i + 1]] = b.T
    _pmap(one, range(auxmol.nbas))
    return out


def q_cond(mol, omega=None):
    """sqrt(max |(ij|ij)|) per shell pair over Cartesian functions (floor 1e-100), as oracle.q_cond over spherical ones."""
    atm, bas, env = O._tables(mol)
    env = env.copy()
    if omega is not None:
        env[8] = omega
    loc = mol.ao_loc_nr(cart=True)
    q = np.zeros((mol.nbas, mol.nbas))
    fn = _fn('int2e_cart')

    def one(i):
        for j in range(i + 1):
            di, dj = loc[i + 1] - loc[i], loc[j + 1] - loc[j]
            b = _call(fn, (di, dj, di, dj), (i, j, i, j), atm, bas, env)
            d = np.abs(np.einsum('abab->ab', b)).max()
            q[i, j] = q[j, i] = max(np.sqrt(d), 1e-100)
    _pmap(one, range(mol.nbas))
    return q


def cholesky_eri(mol, auxmol, lindep=1e-7, omega=None, return_metric=False):
    """cderi[naux', nao(nao+1)/2] over Cartesian functions (pyscf/df/incore.py:129-220: CD, eig fallback :150-158)."""
    if not mol.cart or not auxmol.cart:
        raise ValueError('cart_oracle.cholesky_eri wants Cartesian mol and auxmol')
    saved = mol._env[8]
    if omega is not None:
        mol._env[8] = omega
    try:
        j3c = int3c2e(mol, auxmol)
        j2c = int2c2e(auxmol, omega=mol._env[8])
    finally:
        mol._env[8] = saved
    nao = j3c.shape[0]
    j3c = O.pack_tril(j3c.transpose(2, 0, 1))
    try:
        low = scipy.linalg.cholesky(j2c, lower=True)
        cderi = scipy.linalg.solve_triangular(low, j3c, lower=True)
    except scipy.linalg.LinAlgError:
        w, v = scipy.linalg.eigh(j2c)
        mask = w > lindep
        cderi = (v[:, mask] / np.sqrt(w[mask])).T.dot(j3c)
    cderi = np.ascontiguousarray(cderi)
    return (cderi, nao, j3c, j2c) if return_metric else (cderi, nao)


# ---------------------------------------------------------------------------------------------- one-electron matrices
def _cart_comps(l):
    return [(lx, ly, l - lx - ly) for lx in range(l, -1, -1) for ly in range(l - lx, -1, -1)]


def _shells(mol):
    out = []
    for ib in range(mol.nbas):
        at, l, npr, nct = mol._bas[ib, :4]
        pe, pc = mol._bas[ib, 5], mol._bas[ib, 6]
        r = mol._env[mol._atm[at, 1]:mol._atm[at, 1] + 3]
        out.append((int(l), mol._env[pe:pe + npr].copy(), mol._env[pc:pc + npr * nct].reshape(nct, npr).copy(), r.copy()))
    return out


_GH_X, _GH_W = np.polynomial.hermite.hermgauss(12)   # exact for polynomials of degree <= 23


def _ovlp_1d(i, j, a, b, A, B):
    """int (x-A)^i (x-B)^j exp(-a (x-A)^2 - b (x-B)^2) dx for arrays a, b (exact quadrature)."""
    p = a + b
    P = (a * A + b * B) / p
    pre = np.exp(-a * b / p * (A - B) ** 2) / np.sqrt(p)
    x = _GH_X[:, None, None] / np.sqrt(p) + P
    return pre * np.einsum('k,kab->ab', _GH_W, (x - A) ** i * (x - B) ** j)


def int1e(mol, kind):
    """kind in {'ovlp', 'kin'}: [nao, nao] over Cartesian functions."""
    sh = _shells(mol)
    loc = mol.ao_loc_nr(cart=True)
    nao = int(loc[-1])
    out = np.zeros((nao, nao))
    for i, (la, ea, ca, A) in enumerate(sh):
        for j, (lb, eb, cb, B) in enumerate(sh):
            a, b = ea[:, None], eb[None, :]
            ncb = len(_cart_comps(lb))
            for ia, pa in enumerate(_cart_comps(la)):
                for ib, pb in enumerate(_cart_comps(lb)):
                    S = [_ovlp_1d(pa[x], pb[x], a, b, A[x], B[x]) for x in range(3)]
                    if kind == 'ovlp':
                        prim = S[0] * S[1] * S[2]
                    else:
                        T = []
                        for x in range(3):
                            jx = pb[x]
                            t = 4 * b * b * _ovlp_1d(pa[x], jx + 2, a, b, A[x], B[x]) - 2 * b * (2 * jx + 1) * S[x]
                            if jx >= 2:
                                t = t + jx * (jx - 1) * _ovlp_1d(pa[x], jx - 2, a, b, A[x], B[x])
                            T.append(-0.5 * t)
                        prim = T[0] * S[1] * S[2] + S[0] * T[1] * S[2] + S[0] * S[1] * T[2]
                    blk = ca.dot(prim).dot(cb.T) * _FAC.get(la, 1.0) * _FAC.get(lb, 1.0)   # [nctr_a, nctr_b]
                    na = len(_cart_comps(la))
                    for ci in range(blk.shape[0]):
                        for cj in range(blk.shape[1]):
                            out[loc[i] + ci * na + ia, loc[j] + cj * ncb + ib] = blk[ci, cj]
    return out


def nuc(mol, alpha=1e20):
    """Nuclear attraction -sum_C Z_C (ij|delta_C) over Cartesian functions: int3c2e_cart of the AO pair against an s function
    normalised to unit charge, (alpha/pi)^1.5 exp(-alpha r^2), on each nucleus.  With alpha = 1e20 the smeared charge differs
    from the point charge by O(p/alpha) < 1e-15 relative for every AO exponent p of the basis sets used here."""
    from pyscf_b200 import gto
    atoms = []
    for ia in range(mol.natm):
        atoms.append(('X', tuple(mol._env[mol._atm[ia, 1]:mol._atm[ia, 1] + 3])))
    pt = gto.Mole.__new__(gto.Mole)
    pt.cart = True
    pt._atm = np.zeros((mol.natm, 6), dtype=np.int32)
    env = [0.0] * 20
    bas = []
    for ia, (_, r) in enumerate(atoms):
        pt._atm[ia, 1] = len(env)
        env += list(r)
        bas.append([ia, 0, 1, 1, 0, len(env), len(env) + 1, 0])
        env += [alpha, (alpha / np.pi) ** 1.5 / _FAC[0]]
    pt._bas = np.array(bas, dtype=np.int32)
    pt._env = np.array(env)
    pt.nbas = mol.natm
    pt.ao_loc_nr = lambda cart=True: np.arange(mol.natm + 1)
    saved = mol._env[8]
    mol._env[8] = 0.0
    try:
        j3c = int3c2e(mol, pt)               # [nao, nao, natm]
    finally:
        mol._env[8] = saved
    z = mol._atm[:, 0].astype(np.float64)
    return -np.einsum('ijc,c->ij', j3c, z)


def cart2sph(mol):
    """[nao_cart, nao_sph] block-diagonal map with S_sph = T^T S_cart T: the spherical functions in terms of this module's
    Cartesian ones (identity on s and p, which carry the same factors in both conventions)."""
    lc, ls = mol.ao_loc_nr(cart=True), mol.ao_loc_nr(cart=False)
    T = np.zeros((int(lc[-1]), int(ls[-1])))
    for ib in range(mol.nbas):
        l, nct = int(mol._bas[ib, 1]), int(mol._bas[ib, 3])
        nc, ns = (l + 1) * (l + 2) // 2, 2 * l + 1
        if l < 2:
            blk = np.eye(nc)
        else:
            c = np.zeros(nc * ns)
            O.lib().oracle_c2s(ctypes.c_int(l), O._p(c))
            blk = c.reshape(ns, nc).T
        for k in range(nct):
            T[lc[ib] + k * nc:lc[ib] + (k + 1) * nc, ls[ib] + k * ns:ls[ib] + (k + 1) * ns] = blk
    return T
