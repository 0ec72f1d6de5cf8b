"""The density-fitting 3-center and 2-center Rys kernels class by class against high-precision integrals.

A raw test build (b200jk_df_set_raw_test) runs the shipped b200jk_df_build with the identity as the metric transform, so the
rows of the tensor are the bare (P|mu nu) in the reference layout, and it keeps the assembled metric (P|Q).  Everything else
of the build runs as always: the auxiliary tables, the 3-center batches and the 2-center launch loop, the auxiliary and AO
transforms (spherical or Cartesian), pair screening, host rows and row sharding.  Each element is compared with
tests/eri_ref_df.py (McMurchie-Davidson in long double, with the unit function as the fourth one) and labelled with the kernel
that computed it: j3c_kernel (la lb|lk) with bra class 0..9 for the tensor, (lp s|lq) with bra class pair_class_id(lp, 0)
or 10 for the metric, each in its Coulomb/erf and its erfc (omega < 0) build.

Accuracy bar, as for the 4-center kernels (test_rys_eri.py): |kernel - ref| <= KAPPA * eps * S per (AO shell pair,
auxiliary shell) block of the tensor and per (P, Q) shell block of the metric, S the block maximum of S_abs (the sum of
absolute primitive contributions, carried through |c2s|).  A block with S = 0 (parity zeros: the centres are dyadic, so a
one-centre pair and an auxiliary function on the same centre meet at exactly P - Q = 0) must come out exactly 0.
"""
import ctypes
import os
import re
import time

import numpy as np
import pytest

import eri_ref as R
import eri_ref_df as D
from pyscf_b200 import gto
from pyscf_b200 import lib as b2lib
from test_rys_eri import EPS, KAPPA, PAIR_ID, PAIR_LS, NE, HE, FAR_A, FAR_B, _md_mpmath

pytestmark = pytest.mark.skipif(not R.LONGDOUBLE_OK, reason=R.SKIP_REASON)

# Only in the `far` system, blocks below FLOOR of the system's largest S are held to FLOOR * S_max instead (the horizontal
# recurrence over AO pairs 17.9 bohr apart, as in test_rys_eri.py; measured need in DESIGN.md §4.2).
FLOOR = {'far': 1e-11}

# ---------------------------------------------------------------------------------------------------------------------
# Systems: dyadic centres in bohr.  AO shells on two atoms; auxiliary shells s..g (exponents 0.05 - 1e4) on both of them and,
# in spdf, on a third atom that carries only auxiliary functions.
AO_A = [[0, [1.0e5, 1.0]], [1, [0.9, 1.0]], [2, [0.6, 1.0]], [3, [6.0, 1.0]]]
AO_B = [[0, [0.05, 1.0]], [1, [40.0, 1.0]], [2, [3.0, 1.0]], [3, [0.3, 1.0]]]
AUX_A = [[0, [1.0e4, 1.0]], [1, [0.3, 1.0]], [2, [5.0, 1.0]], [3, [0.7, 1.0]], [4, [2.0, 1.0]]]
AUX_B = [[0, [0.05, 1.0]], [1, [30.0, 1.0]], [2, [0.4, 1.0]], [3, [8.0, 1.0]], [4, [0.15, 1.0]]]
AUX_X = [[0, [1.0, 1.0]], [0, [800.0, 1.0]], [1, [4.0, 1.0]], [2, [0.08, 1.0]], [2, [200.0, 1.0]], [3, [0.5, 1.0]],
         [4, [1.0e4, 1.0]], [4, [0.05, 1.0]]]
# contracted: same-l auxiliary shells of 1, 3 and 5 primitives next to each other (one slot group of j3c_block mixes
# primitive counts), an nctr = 2 shell and a contraction with a zero coefficient
AUX_NE = [[0, [0.5, 1.0]], [0, [30.0, 0.3], [4.0, 0.5], [0.6, 0.4]],
          [0, [2000.0, 0.1], [300.0, 0.2], [40.0, 0.3], [6.0, 0.3], [0.9, 0.2]],
          [1, [1.2, 1.0]], [1, [9.0, 0.4], [2.0, 0.5], [0.4, 0.3]],
          [1, [60.0, 0.1], [15.0, 0.2], [4.0, 0.4], [1.0, 0.3], [0.25, 0.2]],
          [1, [8.0, 0.5], [2.0, 0.0], [0.5, 0.6]],                                     # zero coefficient
          [2, [0.8, 1.0]], [2, [7.0, 0.4], [1.5, 0.5], [0.3, 0.3]],
          [2, [40.0, 0.1], [10.0, 0.2], [3.0, 0.4], [0.9, 0.3], [0.2, 0.2]],
          [2, [5.0, 0.5, 0.1], [1.2, 0.5, -0.6], [0.3, 0.2, 1.0]],                    # nctr = 2
          [3, [1.0, 1.0]], [3, [5.0, 0.5], [1.0, 0.5], [0.2, 0.3]],
          [4, [1.5, 1.0]], [4, [3.0, 0.5], [0.8, 0.5], [0.25, 0.3]],
          [4, [12.0, 0.1], [4.0, 0.3], [1.3, 0.4], [0.45, 0.3], [0.15, 0.1]]]
AUX_HE = [[0, [1.0, 1.0]], [1, [2.0, 1.0]], [2, [1.5, 1.0]], [3, [1.0, 1.0]], [4, [2.5, 1.0]]]
AUX_FA = [[0, [3.0, 1.0]], [1, [0.2, 1.0]], [2, [10.0, 1.0]], [3, [1.0, 1.0]], [4, [0.5, 1.0]]]
AUX_FB = [[0, [0.3, 1.0]], [1, [50.0, 1.0]], [2, [0.6, 1.0]], [3, [4.0, 1.0]], [4, [2.0, 1.0]]]
SYSTEMS = {
    'spdf': (dict(atom='O 0 0 0; C 0.25 -0.5 0.125', basis={'O': AO_A, 'C': AO_B}),
             dict(atom='O 0 0 0; C 0.25 -0.5 0.125; He 2 2 -2', basis={'O': AUX_A, 'C': AUX_B, 'He': AUX_X})),
    'contracted': (dict(atom='Ne 0 0 0; He 1 2 2', basis={'Ne': NE, 'He': HE}),
                   dict(atom='Ne 0 0 0; He 1 2 2', basis={'Ne': AUX_NE, 'He': AUX_HE})),
    'far': (dict(atom='Cl 0 0 0; Ar 0 8 -16', basis={'Cl': FAR_A, 'Ar': FAR_B}),
            dict(atom='Cl 0 0 0; Ar 0 8 -16', basis={'Cl': AUX_FA, 'Ar': AUX_FB})),
}

# ---------------------------------------------------------------------------------------------------------------------
# Kernel labels.  They restate launch decisions of the library: B2_J3C_BRA_CASES (df_classes.cuh) with B2_PAIR_CASES
# (jk_classes.cuh), launch_j3c's switch over the auxiliary l, the metric's bra class in df_build_impl (df.cu) and the SR
# instantiation for omega < 0; test_j3c_labels_match_kernel_sources reads those sources.
BRA_LS = dict(PAIR_LS)
BRA_LS[10] = (4, 0)
LK_MAX = 4
ALL_J3C = sorted((cb, lk) for cb in BRA_LS for lk in range(LK_MAX + 1))
assert len(ALL_J3C) == 55


def metric_bra(lp):
    return 10 if lp == 4 else int(PAIR_ID(lp, 0))


def j3c_name(key):
    (la, lb), lk = BRA_LS[key[0]], key[1]
    return '(%s%s|%s)' % ('spdfg'[la], 'spdfg'[lb], 'spdfg'[lk])


def test_j3c_labels_match_kernel_sources():
    src = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), 'pyscf_b200', 'csrc')
    rd = lambda f: open(os.path.join(src, f)).read()
    jk, dc, df = rd('jk_classes.cuh'), rd('df_classes.cuh'), rd('df.cu')
    cases = re.search(r'#define B2_PAIR_CASES\(X\)\s*\\\s*\n(.*)\n', jk).group(1)
    bra = {int(i): (int(a), int(b)) for i, a, b in re.findall(r'X\((\d+), (\d+), (\d+)\)', cases)}
    extra = re.search(r'#define B2_J3C_BRA_CASES\(X\) B2_PAIR_CASES\(X\)(.*)\n', dc).group(1)
    bra.update({int(i): (int(a), int(b)) for i, a, b in re.findall(r'X\((\d+), (\d+), (\d+)\)', extra)})
    assert bra == BRA_LS, bra
    assert all(int(PAIR_ID(a, b)) == i for i, (a, b) in bra.items() if i < 10)
    body = re.search(r'inline void launch_j3c\(int cb, int lk,.*?\n\}', dc, re.S).group(0)
    assert re.findall(r'case (\d): launch_j3c_lk(\d)\(cb, P, st\)', body) == [(str(l), str(l)) for l in range(LK_MAX + 1)]
    assert 'if (P.omega < 0.0) launch_j3c_kernel<C, true>(P, grid, GC::NT, smem, st);' in dc
    assert 'if (P.omega < 0.0) j3c_block<C, true>(P, bx, by, *sm);' in dc
    assert 'int cb = (lp == 4) ? 10 : pair_class_id(lp, 0);' in df
    assert all(metric_bra(l) == (10 if l == 4 else int(PAIR_ID(l, 0))) for l in range(5))


# ---------------------------------------------------------------------------------------------------------------------
# Reference validation
def test_reference_c2s_g_matches_oracle():
    from oracle import oracle as O
    c = np.zeros(9 * 15)
    O.lib().oracle_c2s(ctypes.c_int(4), O._p(c))
    assert np.abs(c.reshape(9, 15) - R.c2s_matrix(4).astype(np.float64)).max() <= 4 * EPS * np.abs(c).max()


def block_max_axes(t, offs):
    for ax, off in enumerate(offs):
        t = np.maximum.reduceat(t, off[:-1], axis=ax)
    return t


def block_ratio(err, sblk, offs):
    e = block_max_axes(err, offs)
    with np.errstate(divide='ignore', invalid='ignore'):
        return np.where(sblk > 0, e / np.where(sblk > 0, sblk, 1), np.where(e > 0, np.inf, 0.0))


def offsets(segs, cart):
    return np.cumsum([0] + [R.ncart(s.l) if cart else 2 * s.l + 1 for s in segs])


def test_reference_against_oracle():
    """He-Ne/cc-pVDZ with def2-universal-jkfit (g shells, up to 5 primitives): 3-center and 2-center, spherical and
    Cartesian, against the oracle's int3c2e / int2c2e (and their _cart forms) at 1e-13 of S per block."""
    from oracle import oracle as O
    import cart_oracle as CO
    from pyscf_b200.gto.mole import make_auxmol
    mol = gto.M(atom='He 0 0 0; Ne 0.5 1 2', unit='Bohr', basis='ccpvdz')
    aux = make_auxmol(mol, 'def2-universal-jkfit')
    ref = D.DFReference(mol._atm, mol._bas, mol._env, aux._atm, aux._bas, aux._env, prim_cut=0.0)
    v3, s3 = ref.int3c_cart()
    v2, s2 = ref.int2c_cart()
    Ta, Tx = ref.c2s_ao(), ref.c2s_aux()
    worst = 0.0
    for cart in (False, True):
        if cart:
            o3, o2 = CO.int3c2e(mol, aux), CO.int2c2e(aux)
            e3, S3, e2, S2 = v3, s3, v2, s2
        else:
            o3, o2 = O.int3c2e(mol, aux), O.int2c2e(aux)
            e3, S3 = D.to_sph3(v3, Ta, Tx), D.to_sph3(s3, np.abs(Ta), np.abs(Tx))
            e2, S2 = D.to_sph2(v2, Tx), D.to_sph2(s2, np.abs(Tx))
        ao, ax = offsets(ref.segs, cart), offsets(ref.aux, cart)
        e3, S3, e2, S2 = (t.astype(np.float64) for t in (e3, S3, e2, S2))
        r3 = block_ratio(np.abs(e3 - o3), block_max_axes(S3, (ao, ao, ax)), (ao, ao, ax))
        r2 = block_ratio(np.abs(e2 - o2), block_max_axes(S2, (ax, ax)), (ax, ax))
        assert r3.max() <= 1e-13 and r2.max() <= 1e-13, (cart, r3.max(), r2.max())
        worst = max(worst, r3.max(), r2.max())
    print('reference against the oracle: worst block error / S %.2e' % worst)


@pytest.mark.parametrize('ls,exps', [((3, 3, 4), (2.2, 0.8, 1.3)), ((4, 4), (1.7, 0.45))])
def test_reference_primitive_against_mpmath(ls, exps):
    """One (ff|g) and one (g|g) primitive: the 4-center machinery with the unit function against the mpmath
    McMurchie-Davidson of test_rys_eri.py with a zero fourth exponent."""
    if len(ls) == 3:
        centres = ((0, 0, 0), (0.5, -0.25, 1.0), (1.5, 2.0, -0.5))
        seg = [R._Seg(l, np.array(c, dtype=R.LD), np.array([e]), np.array([1.0]), 0) for l, e, c in zip(ls, exps, centres)]
        bra, ket = R._Pair(seg[0], seg[1], 0.0), D.UnitPair(seg[2])
        mls, mexps, mcent = (3, 3, 4, 0), exps + (0.0,), centres + (centres[2],)
    else:
        centres = ((0, 0, 0), (1.5, 2.0, -0.5))
        seg = [R._Seg(l, np.array(c, dtype=R.LD), np.array([e]), np.array([1.0]), 0) for l, e, c in zip(ls, exps, centres)]
        bra, ket = D.UnitPair(seg[0]), D.UnitPair(seg[1])
        mls, mexps, mcent = (4, 0, 4, 0), (exps[0], 0.0, exps[1], 0.0), (centres[0], centres[0], centres[1], centres[1])
    v = R.quartet(bra, ket)[0].astype(np.float64)
    ref = _md_mpmath(mls, mexps, mcent)
    assert np.abs(v - ref).max() <= 8 * EPS * np.abs(ref).max(), np.abs(v - ref).max() / np.abs(ref).max()


# ---------------------------------------------------------------------------------------------------------------------
# Reference cache (module scope, per system and operator) and the raw builds
_REF = {}


def mols(name, cart=False):
    ao, aux = SYSTEMS[name]
    return gto.M(unit='Bohr', cart=cart, **ao), gto.M(unit='Bohr', **aux)


def reference(name, omega):
    """(DFReference, v3, S3, v2, S2, {n_roots: x}) in Cartesian functions, cached."""
    key = (name, omega)
    if key not in _REF:
        mol, aux = mols(name)
        ref = D.DFReference(mol._atm, mol._bas, mol._env, aux._atm, aux._bas, aux._env)
        xlog = {}
        v3, s3 = ref.int3c_cart(omega, xlog)
        v2, s2 = ref.int2c_cart(omega, xlog)
        _REF[key] = (ref, v3, s3, v2, s2, {n: np.concatenate(x) for n, x in xlog.items()})
    return _REF[key]


def raw_build(lib, name, omega, cart=False, device_rows=-1, shard=None, pair_tol=0.0, raw=True, h=None):
    """Build on a (new) handle and return (handle, local tensor rows [nrow, npair], metric or None)."""
    mol, aux = mols(name, cart)
    if h is None:
        h = b2lib.Handle(mol._atm, mol._bas, mol._env, libpath=lib, cart=cart)
    if shard is not None:
        h.check(h.lib.b200jk_set_shard(h._h, *shard), 'b200jk_set_shard')
    h.check(h.lib.b200jk_df_set_device_rows(h._h, int(device_rows)), 'b200jk_df_set_device_rows')
    h.check(h.lib.b200jk_df_set_pair_tol(h._h, float(pair_tol)), 'b200jk_df_set_pair_tol')
    h.check(h.lib.b200jk_df_set_raw_test(h._h, int(raw)), 'b200jk_df_set_raw_test')
    atm, bas = (np.ascontiguousarray(a, dtype=np.int32) for a in (aux._atm, aux._bas))
    env = np.ascontiguousarray(aux._env, dtype=np.float64)
    h.check(h.lib.b200jk_df_build(h._h, b2lib.iptr(atm), len(atm), b2lib.iptr(bas), len(bas), b2lib.dptr(env), len(env),
                                  float(omega), 1e-7), 'b200jk_df_build')
    return (h,) + read_back(h, raw)


def read_back(h, raw):
    row0, nrow, naux = ctypes.c_int(0), ctypes.c_int(0), ctypes.c_int(0)
    h.check(h.lib.b200jk_df_local_rows(h._h, ctypes.byref(row0), ctypes.byref(nrow)), 'b200jk_df_local_rows')
    h.check(h.lib.b200jk_df_naux(h._h, ctypes.byref(naux)), 'b200jk_df_naux')
    ncol, npair = ctypes.c_int64(0), ctypes.c_int64(0)
    h.check(h.lib.b200jk_df_pair_stats(h._h, ctypes.byref(ncol), ctypes.byref(npair)), 'b200jk_df_pair_stats')
    t = np.empty((nrow.value, npair.value))
    h.check(h.lib.b200jk_df_get_cderi(h._h, b2lib.dptr(t), 0, nrow.value), 'b200jk_df_get_cderi')
    j2c = None
    if raw:
        j2c = np.empty((naux.value, naux.value))
        h.check(h.lib.b200jk_df_get_metric_test(h._h, b2lib.dptr(j2c), naux.value), 'b200jk_df_get_metric_test')
    return t, j2c


def unpack(t, nao):
    """[naux, npair] packed rows -> [naux, nao, nao]."""
    mu, nu = np.tril_indices(nao)
    out = np.zeros((t.shape[0], nao, nao))
    out[:, mu, nu] = t
    out[:, nu, mu] = t
    return out


class Tally:
    """Largest error / S per kernel instantiation (bra class, auxiliary l, SR), and the coverage of the runs."""

    def __init__(self):
        self.worst = {}
        self.xs = {}

    def expected(self, name, omega, cart):
        """Reference in the handle's convention: (v3[naux, nao, nao], S3 blocks, v2, S2 blocks, offsets, labels)."""
        ref, v3, s3, v2, s2, xlog = reference(name, omega)
        if cart:
            e3, S3, e2, S2 = v3, s3, v2, s2
        else:
            Ta, Tx = ref.c2s_ao(), ref.c2s_aux()
            e3, S3 = D.to_sph3(v3, Ta, Tx), D.to_sph3(s3, np.abs(Ta), np.abs(Tx))
            e2, S2 = D.to_sph2(v2, Tx), D.to_sph2(s2, np.abs(Tx))
        e3, S3, e2, S2 = (np.ascontiguousarray(t.astype(np.float64)) for t in (e3, S3, e2, S2))
        return ref, e3.transpose(2, 0, 1), S3.transpose(2, 0, 1), e2, S2, xlog

    def add(self, label, name, omega, cart, t, j2c, rows=None, floor=None):
        """t: tensor rows [rows] (all rows when None) of a raw build, j2c: its metric (or None)."""
        ref, e3, S3, e2, S2, xlog = self.expected(name, omega, cart)
        floor = FLOOR.get(name, 0.0) if floor is None else floor
        ao, ax = offsets(ref.segs, cart), offsets(ref.aux, cart)
        nao = int(ao[-1])
        lao = np.array([s.l for s in ref.segs])
        lax = np.array([s.l for s in ref.aux])
        sr = omega < 0
        bad = []
        if rows is None:
            rows = np.arange(e3.shape[0])
        assert t.shape == (len(rows), nao * (nao + 1) // 2), t.shape
        # the tensor: blocks (auxiliary shell, AO shell, AO shell); rows this build does not hold (another shard's) count as
        # exact, and auxiliary shells without a held row are skipped
        k3 = e3.copy()
        k3[rows] = unpack(t, nao)
        present = np.zeros(e3.shape[0], dtype=bool)
        present[rows] = True
        offs3 = (ax, ao, ao)
        sb = block_max_axes(S3, offs3)
        if floor:
            sb = np.where(sb > 0, np.maximum(sb, floor * sb.max()), 0.0)
        r3 = block_ratio(np.abs(k3 - e3), sb, offs3) / EPS
        have = np.maximum.reduceat(present.astype(float), ax[:-1]) > 0
        cb3 = PAIR_ID(lao[:, None], lao[None, :])
        for key in ALL_J3C:
            m = (cb3[None] == key[0]) & (lax[:, None, None] == key[1]) & have[:, None, None]
            if key[0] < 10 and m.any():
                self._note(key, sr, r3[m], r3, m, label, 'tensor', bad)
        if j2c is not None:
            offs2 = (ax, ax)
            sb2 = block_max_axes(S2, offs2)
            if floor:
                sb2 = np.where(sb2 > 0, np.maximum(sb2, floor * sb2.max()), 0.0)
            r2 = block_ratio(np.abs(j2c - e2), sb2, offs2) / EPS
            # element [row Q][column P] comes from the launch with bra P (column) and ket Q (row)
            bra = np.array([metric_bra(l) for l in lax])
            for key in ALL_J3C:
                m = (bra[None, :] == key[0]) & (lax[:, None] == key[1])
                if m.any():
                    self._note(key, sr, r2[m], r2, m, label, 'metric', bad)
        for n, x in xlog.items():
            self.xs.setdefault(n, []).append(x)
        ok3 = r3[np.isfinite(r3)]
        print('%-40s worst %.1f eps' % (label, ok3.max() if ok3.size else 0.0), flush=True)
        assert not bad, '\n'.join(bad)

    def _note(self, key, sr, r, full, mask, label, what, bad):
        k = (key, sr)
        self.worst[k] = max(self.worst.get(k, 0.0), float(r.max()))
        if r.max() > KAPPA:
            q = np.argwhere(mask & (full == r.max()))[0]
            bad.append('j3c_kernel %s%s [%s, %s]: block %s, error/S = %.3g eps, bar %d eps' % (
                j3c_name(key), ' SR' if sr else '', label, what, tuple(int(v) for v in q), r.max(), KAPPA))

    def report(self, what):
        print('%s: largest error / S per j3c_kernel instantiation, in units of eps (omega >= 0, omega < 0); bar %d eps'
              % (what, KAPPA))
        for key in ALL_J3C:
            print('  %-8s %7.1f %7.1f' % (j3c_name(key), self.worst.get((key, False), -1), self.worst.get((key, True), -1)))

    def check_coverage(self, xs=True):
        for sr in (False, True):
            missing = [j3c_name(k) for k in ALL_J3C if (k, sr) not in self.worst]
            assert not missing, 'instantiations never reached (SR=%s): %s' % (sr, missing)
        if not xs:
            return
        counts = {}
        for n in range(1, 7):
            x = np.concatenate(self.xs.get(n, [np.zeros(0)]))
            counts[n] = (int((x == 0).sum()), int(((x > 0) & (x < 100)).sum()), int((x >= 100).sum()))
            assert all(c > 0 for c in counts[n]), 'n=%d: primitive products at x = 0, 0 < x < 100, x >= 100: %s' % (n, counts[n])
        print('x per root count n (x = 0, 0 < x < 100, x >= 100):', counts)


def run_case(tally, lib, name, omega, cart=False):
    t0 = time.time()
    h, t, j2c = raw_build(lib, name, omega, cart)
    h.close()
    tally.add('%s%s omega=%g (%.0f s)' % (name, ' cart' if cart else '', omega, time.time() - t0), name, omega, cart, t, j2c)
    return t


def check_far_cut():
    """far has an AO pair all of whose primitive pairs fall under PRIM_CUT (the s pair of exponents 2 and 500, 17.9 bohr
    apart): its reference block is exactly 0 with S = 0, so Tally.add holds the kernel's columns to exactly 0."""
    ref = reference('far', 0.0)[0]
    assert any(p.nprim == 0 and np.any(p.A.r != p.B.r) for p in ref.pairs.values())


def check_contracted_aux():
    """The contracted auxiliary basis has same-l shells of 1, 3 and 5 primitives in a row, an nctr = 2 shell and a zero
    coefficient, as the layout of build_aux sees them."""
    ref = reference('contracted', 0.0)[0]
    _, aux = mols('contracted')
    assert any(b[3] == 2 for b in aux._bas)
    assert any((aux._env[b[6]:b[6] + b[2] * b[3]] == 0).any() for b in aux._bas)
    per_l = {}
    for s in ref.aux:
        per_l.setdefault(s.l, []).append(len(s.e))
    assert {1, 3, 5} <= set(per_l[0]) and {1, 3, 5} <= set(per_l[2]) and {1, 3, 5} <= set(per_l[4]), per_l


# ---------------------------------------------------------------------------------------------------------------------
# Layout legs on `contracted`, omega = 0: host rows, two shard ranks and pair screening, against the same reference
def q_cond(name, cart, omega=0.0):
    """q = sqrt(max over the pair's functions of |(ab|ab)|) per segment pair (CVHFnr_int2e_q_cond), from eri_ref."""
    ref = reference(name, omega)[0]
    q = {}
    for (i, j), p in ref.pairs.items():
        v = R.quartet(p, p, omega)[0]
        if not cart:
            T = np.kron(R.c2s_matrix(p.la), R.c2s_matrix(p.lb))
            v = T.dot(v).dot(T.T)
        q[i, j] = float(np.sqrt(np.abs(np.diag(v.astype(np.float64))).max())) if p.nprim else 0.0
    return q


def check_layouts(lib, cart=False):
    name, omega = 'contracted', 0.0
    tally = Tally()
    h, full, j2c = raw_build(lib, name, omega, cart)
    h.close()
    tally.add('%s%s dense' % (name, ' cart' if cart else ''), name, omega, cart, full, j2c)
    naux = full.shape[0]
    # host rows
    h, t, _ = raw_build(lib, name, omega, cart, device_rows=naux // 3)
    n_dev, n_host = ctypes.c_int(0), ctypes.c_int(0)
    h.check(h.lib.b200jk_df_row_split(h._h, ctypes.byref(n_dev), ctypes.byref(n_host)), 'b200jk_df_row_split')
    h.close()
    assert n_dev.value == naux // 3 and n_host.value == naux - naux // 3
    tally.add('%s host rows %d+%d' % (name, n_dev.value, n_host.value), name, omega, cart, t, None)
    assert np.array_equal(t, full)
    # two shard ranks: the local rows concatenated
    parts = []
    for r in range(2):
        h, t, _ = raw_build(lib, name, omega, cart, shard=(r, 2))
        h.close()
        assert t.shape[0] == naux * (r + 1) // 2 - naux * r // 2
        tally.add('%s shard %d/2' % (name, r), name, omega, cart, t, None, rows=np.arange(naux * r // 2, naux * (r + 1) // 2))
        parts.append(t)
    assert np.array_equal(np.vstack(parts), full)
    # pair screening with pair_tol between two well-separated Schwarz bounds
    ref = reference(name, omega)[0]
    q = q_cond(name, cart)
    qs = np.array(sorted(v for v in q.values() if v > 0))
    # the largest ratio of neighbouring bounds (2.3 on contracted); tol in its geometric middle sits a factor > 1.4 from
    # either bound, far beyond the rounding of the library's own q
    gap = int(np.argmax(qs[1:] / qs[:-1]))
    assert qs[gap + 1] / qs[gap] > 2, qs
    tol = float(np.sqrt(qs[gap] * qs[gap + 1]))
    h, t, _ = raw_build(lib, name, omega, cart, pair_tol=tol)
    ncol = ctypes.c_int64(0); npair = ctypes.c_int64(0)
    h.check(h.lib.b200jk_df_pair_stats(h._h, ctypes.byref(ncol), ctypes.byref(npair)), 'b200jk_df_pair_stats')
    h.close()
    ao = offsets(ref.segs, cart)
    nao = int(ao[-1])
    seg = np.searchsorted(ao, np.arange(nao), side='right') - 1
    mu, nu = np.tril_indices(nao)
    kept_pairs = {k for k, v in q.items() if v >= tol}
    kept = np.array([(seg[a], seg[b]) in kept_pairs or (seg[b], seg[a]) in kept_pairs for a, b in zip(mu, nu)])
    assert 0 < kept.sum() < len(kept) and ncol.value == kept.sum(), (ncol.value, kept.sum())
    # kept columns: the dense build's (checked against the reference above) bit for bit; dropped ones exactly 0
    assert np.array_equal(t[:, kept], full[:, kept])
    assert not t[:, ~kept].any()
    print('%s pair_tol=%.2e: %d of %d columns kept' % (name, tol, kept.sum(), len(kept)))
    return tally


# ---------------------------------------------------------------------------------------------------------------------
# CPU emulation
def test_raw_mode_switches_off(emu_lib):
    """Raw mode is off by default and leaves nothing behind: raw then non-raw on one handle gives a fresh handle's tensor
    bit for bit (H2O/weigend); a raw handle has no metric factor for the integral-direct J and a non-raw one no metric copy."""
    from conftest import H2O
    from pyscf_b200.gto.mole import make_auxmol
    mol = gto.M(atom=H2O, basis='ccpvdz')
    aux = make_auxmol(mol, 'weigend')
    atm, bas = (np.ascontiguousarray(a, dtype=np.int32) for a in (aux._atm, aux._bas))
    env = np.ascontiguousarray(aux._env, dtype=np.float64)

    def build(h, raw=None):
        if raw is not None:
            h.check(h.lib.b200jk_df_set_raw_test(h._h, raw), 'b200jk_df_set_raw_test')
        h.check(h.lib.b200jk_df_build(h._h, b2lib.iptr(atm), len(atm), b2lib.iptr(bas), len(bas), b2lib.dptr(env),
                                      len(env), 0.0, 1e-7), 'b200jk_df_build')
        return read_back(h, False)[0]

    fresh = b2lib.Handle(mol._atm, mol._bas, mol._env, libpath=emu_lib)
    ref = build(fresh)
    j2c = np.empty((ref.shape[0],) * 2)
    assert fresh.lib.b200jk_df_get_metric_test(fresh._h, b2lib.dptr(j2c), ref.shape[0]) != 0
    fresh.close()
    h = b2lib.Handle(mol._atm, mol._bas, mol._env, libpath=emu_lib)
    raw = build(h, 1)
    assert raw.shape == ref.shape and not np.array_equal(raw, ref)
    dm = np.eye(mol.nao)
    vj = np.empty_like(dm)
    assert h.lib.b200jk_df_direct_j(h._h, b2lib.dptr(dm), 1, mol.nao, b2lib.dptr(vj)) != 0
    again = build(h, 0)
    h.close()
    assert np.array_equal(again, ref)


OMEGAS = (0.0, 0.35, 8.0, -0.4)


def test_df_classes_emulated(emu_lib):
    """spdf and far with all four operators, spherical and Cartesian: every instantiation in both builds, and x on both
    sides of 100 for n = 1..6."""
    tally = Tally()
    for name in ('spdf', 'far'):
        for cart in (False, True):
            for omega in OMEGAS:
                run_case(tally, emu_lib, name, omega, cart)
    tally.report('CPU emulation')
    tally.check_coverage()
    check_far_cut()


def test_df_contracted_emulated(emu_lib):
    """contracted: mixed primitive counts in one slot group, nctr = 2, zero coefficients; all four operators, spherical and
    Cartesian."""
    check_contracted_aux()
    tally = Tally()
    for cart in (False, True):
        for omega in OMEGAS:
            run_case(tally, emu_lib, 'contracted', omega, cart)
    tally.report('CPU emulation, contracted')
    tally.check_coverage(xs=False)


def test_df_layouts_emulated(emu_lib):
    check_layouts(emu_lib).report('CPU emulation, contracted layouts')


def test_df_experimental_layouts_emulated(emu_lib_experimental):
    """The experimental lane layouts (B2_PBMAX / B2_PPW reach j3c_block through GroupCfg) on spdf and contracted."""
    tally = Tally()
    for omega in (0.0, -0.4):
        run_case(tally, emu_lib_experimental, 'spdf', omega)
    run_case(tally, emu_lib_experimental, 'contracted', 0.0)
    tally.report('CPU emulation, experimental layouts')


# ---------------------------------------------------------------------------------------------------------------------
# H100
DEVICE_CASES = {
    'spdf': [(0.0, False), (0.35, False), (8.0, False), (-0.4, False), (8.0, True), (-0.4, True)],
    'far': [(0.0, False), (0.35, False), (8.0, False), (-0.4, False)],
    'contracted': [(0.0, False), (-0.4, False), (0.35, True), (-0.4, True)],
}


@pytest.mark.gpu
@pytest.mark.parametrize('case', list(DEVICE_CASES))
def test_df_classes_device(case):
    tally = Tally()
    for omega, cart in DEVICE_CASES[case]:
        run_case(tally, None, case, omega, cart)
    tally.report('H100, %s' % case)
    if case == 'spdf':
        tally.check_coverage()
    if case == 'contracted':
        check_contracted_aux()


@pytest.mark.gpu
def test_df_layouts_device():
    check_layouts(None).report('H100, contracted layouts')
