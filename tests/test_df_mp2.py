"""DF-MP2 energies and amplitudes on the GPU (pyscf_b200.dfmp2: b200jk_df_mp2, df_mp2.cuh) — the DFRMP2 / DFUMP2 kernels of
pyscf/mp/dfmp2.py:39-121 and dfump2.py:38-166.

The model is a numpy restatement of MP2_contract_d / MP2_OS_contract_d (pyscf/lib/mp/mp2.c:89-275) on a tensor: pair by pair
V = iaL[i] jbL[j]^T, t = V / D, ed += fac V.t, ex -= fac V^T.t, with the pair factor of _MP2_gen_jobs.  It is pinned to the
reference's own answers for H2O/cc-pVDZ (pyscf/mp/test/test_dfmp2.py) on the oracle's tensors, and the kernel is checked
against it on the tensor read back with DF.loop(): |de_ss|, |de_os| <= 1e-10 Eh and t2 element-wise <= 1e-12 max|t2|.  The CPU
emulation runs the same CTA code (tiling, the two-tile epilogue, edge tiles, the reduction) on a host model of the fragments;
the GPU tier repeats the cases on sm_90a and adds benzene/cc-pVDZ in full and C60/def2-SVP against DF.ao2mo."""
import json
import os

import numpy as np
import pytest
import scipy.linalg

from pyscf_b200 import dfmp2, gto
from pyscf_b200.df import DF
from pyscf_b200.gto.mole import geometry, make_auxmol
from oracle import oracle as O

H2O = 'O 0 0 0; H 0 -0.757 0.587; H 0 0.757 0.587'
_GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), 'golden')


def _ri_basis():
    """H and O shells of cc-pVDZ-RI (tools/make_fixture_mp2fit.py), the MP2-fit basis the reference picks for cc-pVDZ."""
    with open(os.path.join(_GOLDEN, 'basis_cc-pvdz-ri.json')) as f:
        return json.load(f)


# ---- the model ----------------------------------------------------------------------------------------------------------------

def _unpack(B, nao):
    out = np.zeros((len(B), nao, nao))
    i, j = np.tril_indices(nao)
    out[:, i, j] = B
    out[:, j, i] = B
    return out


def _ovL(B, nao, co, cv):
    """iaL[i, a, P] = C_occ[:, i]^T B_P C_vir[:, a]."""
    return np.einsum('pmn,mi,na->iap', _unpack(B, nao), co, cv, optimize=True)


def _contract(iaL, jbL, eo_i, eo_j, ev_a, ev_b, same_spin, t2_ex=False, with_t2=True):
    """MP2_contract_d (same_spin, s2symm = 1) / MP2_OS_contract_d: (ed, ex, t2)."""
    ni, nj = len(iaL), len(jbL)
    moevv = ev_a[:, None] + ev_b[None, :]
    ed = ex = 0.0
    t2 = np.zeros((ni, nj, len(ev_a), len(ev_b))) if with_t2 else None
    for i in range(ni):
        for j in range(i + 1 if same_spin else nj):
            fac = (1.0 if i == j else 2.0) if same_spin else 1.0
            vab = iaL[i] @ jbL[j].T
            tab = vab / (eo_i[i] + eo_j[j] - moevv)
            ed += np.sum(vab * tab) * fac
            if same_spin:
                ex -= np.sum(vab.T * tab) * fac
                if t2_ex:
                    tab = tab - tab.T
            if with_t2:
                t2[i, j] = tab
                if same_spin and i != j:
                    t2[j, i] = tab.T
    return ed, ex, t2


def model_rmp2(B, nao, co, cv, eo, ev):
    """(e_ss, e_os, t2) of dfmp2.kernel (dfmp2.py:109-119)."""
    if co.shape[1] == 0 or cv.shape[1] == 0:
        return 0.0, 0.0, np.zeros((co.shape[1],) * 2 + (cv.shape[1],) * 2)
    L = _ovL(B, nao, co, cv)
    ed, ex, t2 = _contract(L, L, eo, eo, ev, ev, True)
    return ed + ex, ed, t2


def model_ump2(B, nao, cos, cvs, eos, evs):
    """(e_ss, e_os, (t2aa, t2ab, t2bb)) of dfump2.kernel (dfump2.py:119,154,164)."""
    no = [c.shape[1] for c in cos]
    nv = [c.shape[1] for c in cvs]
    L = [_ovL(B, nao, cos[s], cvs[s]) if no[s] and nv[s] else None for s in (0, 1)]
    e_ss = 0.0
    t2 = [np.zeros((no[0], no[0], nv[0], nv[0])), np.zeros((no[0], no[1], nv[0], nv[1])), np.zeros((no[1], no[1], nv[1], nv[1]))]
    for s in (0, 1):
        if L[s] is not None:
            ed, ex, t2[2 * s] = _contract(L[s], L[s], eos[s], eos[s], evs[s], evs[s], True, t2_ex=True)
            e_ss += (ed + ex) * 0.5
    e_os = 0.0
    if L[0] is not None and L[1] is not None:
        e_os, _, t2[1] = _contract(L[0], L[1], eos[0], eos[1], evs[0], evs[1], False)
    return e_ss, e_os, tuple(t2)


# ---- SCF to the reference's convergence ----------------------------------------------------------------------------------------

def _scf(mol, get_jk):
    """Closed-shell SCF with DIIS, converged to an orbital gradient of 1e-10 (the reference tests use conv_tol = 1e-12)."""
    s = O.int1e(mol, 'ovlp')
    hcore = O.int1e(mol, 'kin') + O.int1e(mol, 'nuc')
    nocc = mol.nelectron // 2
    e, c = scipy.linalg.eigh(hcore, s)
    fs, es = [], []
    for it in range(100):
        dm = 2.0 * c[:, :nocc] @ c[:, :nocc].T
        vj, vk = get_jk(dm)
        f = hcore + vj - 0.5 * vk
        err = f @ dm @ s
        err = err - err.T
        if abs(err).max() < 1e-10:
            break
        fs, es = (fs + [f])[-8:], (es + [err])[-8:]
        n = len(fs)
        b = -np.ones((n + 1, n + 1))
        b[n, n] = 0.0
        b[:n, :n] = [[np.vdot(x, y) for y in es] for x in es]
        w = np.linalg.solve(b, np.r_[np.zeros(n), -1.0])[:n]
        e, c = scipy.linalg.eigh(sum(wi * fi for wi, fi in zip(w, fs)), s)
    else:
        raise AssertionError('SCF did not converge')
    e, c = scipy.linalg.eigh(f, s)
    return e, c


def _uhf(mol, nel, guess):
    """UHF with DIIS from the orbitals `guess` for both spins, converged to an orbital gradient of 1e-10; nel = (n_alpha, n_beta)."""
    s = O.int1e(mol, 'ovlp')
    hcore = O.int1e(mol, 'kin') + O.int1e(mol, 'nuc')
    cs = [guess, guess]
    fs, es = [], []
    for it in range(100):
        dms = np.array([c[:, :n] @ c[:, :n].T for c, n in zip(cs, nel)])
        vj, vk = O.get_jk(mol, dms)
        f = np.array([hcore + vj[0] + vj[1] - vk[k] for k in (0, 1)])
        err = np.concatenate([(f[k] @ dms[k] @ s - s @ dms[k] @ f[k]).ravel() for k in (0, 1)])
        if abs(err).max() < 1e-10:
            break
        fs, es = (fs + [f])[-8:], (es + [err])[-8:]
        n = len(fs)
        b = -np.ones((n + 1, n + 1))
        b[n, n] = 0.0
        b[:n, :n] = [[x @ y for y in es] for x in es]
        w = np.linalg.solve(b, np.r_[np.zeros(n), -1.0])[:n]
        fb = sum(wi * fi for wi, fi in zip(w, fs))
        cs = [scipy.linalg.eigh(fb[k], s)[1] for k in (0, 1)]
    else:
        raise AssertionError('UHF did not converge')
    return [scipy.linalg.eigh(f[k], s) for k in (0, 1)]


_CACHE = {}


def _h2o_scf():
    """H2O/cc-pVDZ RHF orbitals from the oracle's 4-center J/K (mf of pyscf/mp/test/test_dfmp2.py:36-38)."""
    if 'h2o' not in _CACHE:
        mol = gto.M(atom=H2O, basis='cc-pvdz')
        _CACHE['h2o'] = (mol,) + _scf(mol, lambda dm: O.get_jk(mol, dm))
    return _CACHE['h2o']


def _split(mo, e, nocc, frozen):
    """_mo_splitter (pyscf/mp/mp2.py:206-215): active occupied and virtual coefficients and energies."""
    act = np.ones(mo.shape[1], dtype=bool)
    act[list(frozen)] = False
    occ = np.arange(mo.shape[1]) < nocc
    return mo[:, occ & act], mo[:, ~occ & act], e[occ & act], e[~occ & act]


# ---- the model against the reference (CPU, oracle only) -----------------------------------------------------------------------

@pytest.mark.parametrize('frozen,e_ref', [((), -0.20400482102770082),          # test_dfmp2.py:63
                                          ((0, 1, 5), -0.13844381496025246),   # :73
                                          ((0,), -0.20166760413156876)])       # :81
def test_model_reference_pins(frozen, e_ref):
    """DFMP2(mf) with mf an RHF from 4-center J/K: the MP2-fit tensor is cc-pVDZ-RI (make_auxbasis(mp2fit=True))."""
    mol, e, c = _h2o_scf()
    B, nao = O.cholesky_eri(mol, make_auxmol(mol, _ri_basis()))
    co, cv, eo, ev = _split(c, e, mol.nelectron // 2, frozen)
    e_ss, e_os, _ = model_rmp2(B, nao, co, cv, eo, ev)
    assert abs(e_ss + e_os - e_ref) < 5e-9, (e_ss + e_os, e_ref)


def test_model_reference_pin_jkfit_scf():
    """test_dfmp2.py:104: the SCF fitted with cc-pVDZ-JKFIT, MP2 with cc-pVDZ-RI."""
    mol = gto.M(atom=H2O, basis='cc-pvdz')
    Bjk, nao = O.cholesky_eri(mol, make_auxmol(mol, 'cc-pvdz-jkfit'))
    e, c = _scf(mol, lambda dm: O.df_get_jk(Bjk, nao, dm))
    B, _ = O.cholesky_eri(mol, make_auxmol(mol, _ri_basis()))
    co, cv, eo, ev = _split(c, e, mol.nelectron // 2, ())
    e_ss, e_os, _ = model_rmp2(B, nao, co, cv, eo, ev)
    assert abs(e_ss + e_os + 0.20399004345216082) < 5e-9, e_ss + e_os


@pytest.mark.parametrize('frozen,e_ref', [(((), ()), -0.15321910903780497),          # test_dfump2.py:60
                                          (((0, 1, 5), (1,)), -0.09397152054462676)])  # :70
def test_model_reference_pins_ump2(frozen, e_ref):
    """DFUMP2(mf) with mf a UHF of H2O+ (doublet) from 4-center J/K, started from the neutral RHF orbitals; cc-pVDZ-RI tensor."""
    mol, e, c = _h2o_scf()
    nel = (5, 4)
    orbs = _uhf(mol, nel, c)
    B, nao = O.cholesky_eri(mol, make_auxmol(mol, _ri_basis()))
    sp = [_split(orbs[k][1], orbs[k][0], nel[k], frozen[k]) for k in (0, 1)]
    e_ss, e_os, _ = model_ump2(B, nao, [x[0] for x in sp], [x[1] for x in sp], [x[2] for x in sp], [x[3] for x in sp])
    assert abs(e_ss + e_os - e_ref) < 5e-9, (e_ss + e_os, e_ref)


# ---- the kernel against the model (emulated, and on sm_90a) -----------------------------------------------------------------

def _check_r(d, B, co, cv, eo, ev, with_t2=True):
    e, t2 = dfmp2.kernel(d, co, cv, eo, ev, with_t2=with_t2)
    e_ss, e_os, t2m = model_rmp2(B, d.nao, co, cv, eo, ev)
    assert isinstance(e, float) and e == e.e_corr_ss + e.e_corr_os
    assert abs(e.e_corr_ss - e_ss) <= 1e-10 and abs(e.e_corr_os - e_os) <= 1e-10, (e.e_corr_ss - e_ss, e.e_corr_os - e_os)
    if with_t2:
        assert t2.shape == t2m.shape
        if t2.size:
            assert abs(t2 - t2m).max() <= 1e-12 * abs(t2m).max(), abs(t2 - t2m).max() / abs(t2m).max()
    else:
        assert t2 is None
    return e, t2


def _check_u(d, B, cos, cvs, eos, evs):
    e, t2 = dfmp2.ukernel(d, cos, cvs, eos, evs, with_t2=True)
    e_ss, e_os, t2m = model_ump2(B, d.nao, cos, cvs, eos, evs)
    assert abs(e.e_corr_ss - e_ss) <= 1e-10 and abs(e.e_corr_os - e_os) <= 1e-10, (e.e_corr_ss - e_ss, e.e_corr_os - e_os)
    assert len(t2) == 3
    for got, want in zip(t2, t2m):
        assert got.shape == want.shape
        if want.size:
            assert abs(got - want).max() <= 1e-12 * abs(want).max()
    return e, t2


def _set_tile(d, rows):
    h = d._handle
    h.check(h.lib.b200jk_df_set_ao2mo_tile(h._h, int(rows)), 'b200jk_df_set_ao2mo_tile')


def _h2o_df(libpath):
    key = ('df', libpath)
    if key not in _CACHE:
        mol, e, c = _h2o_scf()
        d = DF(mol, _ri_basis(), libpath=libpath).build()
        _CACHE[key] = (mol, e, c, d, d._cderi)
    return _CACHE[key]


def _h2o_cases(libpath):
    """RMP2 with and without frozen orbitals, nocc = 1, no virtual orbitals; UMP2 with different alpha / beta sets, alpha = beta,
    a spin without virtual orbitals; determinism, host rows, bands of t2."""
    mol, e, c, d, B = _h2o_df(libpath)
    nocc = mol.nelectron // 2
    full = _check_r(d, B, *_split(c, e, nocc, ()))
    _check_r(d, B, *_split(c, e, nocc, (0, 1, 5)))
    _check_r(d, B, c[:, 4:5], c[:, 5:], e[4:5], e[5:])                     # nocc = 1
    e0, t0 = _check_r(d, B, c[:, :nocc], c[:, :0], e[:nocc], e[:0])          # no virtual orbitals: exactly 0
    assert e0 == 0.0 and e0.e_corr_ss == 0.0 and e0.e_corr_os == 0.0 and t0.shape == (nocc, nocc, 0, 0)
    # determinism, and the energy does not depend on with_t2
    again = dfmp2.kernel(d, c[:, :nocc], c[:, nocc:], e[:nocc], e[nocc:], with_t2=False)[0]
    assert (again, again.e_corr_ss, again.e_corr_os) == (full[0], full[0].e_corr_ss, full[0].e_corr_os)

    # UMP2: beta = a rotated set with one electron fewer (the shape of H2O+), shifted energies
    rng = np.random.RandomState(3)
    rot = scipy.linalg.expm(0.05 * (lambda a: a - a.T)(rng.standard_normal((c.shape[1],) * 2)))
    cb, eb = c @ rot, e + 0.01 * rng.standard_normal(len(e))
    cos, cvs = [c[:, :nocc], cb[:, :nocc - 1]], [c[:, nocc:], cb[:, nocc - 1:]]
    eos, evs = [e[:nocc], eb[:nocc - 1]], [e[nocc:], eb[nocc - 1:]]
    _check_u(d, B, cos, cvs, eos, evs)
    _check_u(d, B, [c[:, :nocc], cb[:, :nocc]], [c[:, nocc:], cb[:, :0]], [e[:nocc], eb[:nocc]], [e[nocc:], eb[:0]])
    # alpha = beta reproduces RMP2
    eu, tu = dfmp2.ukernel(d, [c[:, :nocc]] * 2, [c[:, nocc:]] * 2, [e[:nocc]] * 2, [e[nocc:]] * 2, with_t2=True)
    er = full[0]
    assert abs(eu.e_corr_ss - er.e_corr_ss) <= 1e-12 and abs(eu.e_corr_os - er.e_corr_os) <= 1e-12
    assert abs(tu[1] - full[1]).max() <= 1e-12 * abs(full[1]).max()

    # several bands of t2 through the pipeline, and half of the rows on the host: bit for bit
    for rows in (1, 4):
        _set_tile(d, rows)
        try:
            banded = dfmp2.kernel(d, c[:, :nocc], c[:, nocc:], e[:nocc], e[nocc:], with_t2=True)
            ub = dfmp2.ukernel(d, cos, cvs, eos, evs, with_t2=True)
        finally:
            _set_tile(d, -1)
        assert banded[0] == full[0] and banded[0].e_corr_ss == full[0].e_corr_ss and np.array_equal(banded[1], full[1]), rows
        uref = dfmp2.ukernel(d, cos, cvs, eos, evs, with_t2=True)
        assert ub[0] == uref[0] and all(np.array_equal(a, b) for a, b in zip(ub[1], uref[1]))
    naux = d.get_naoaux()
    hd = DF(mol, _ri_basis(), libpath=libpath).set_device_rows(naux // 2).build()
    try:
        assert hd.row_split() == (naux // 2, naux - naux // 2)
        hr = dfmp2.kernel(hd, c[:, :nocc], c[:, nocc:], e[:nocc], e[nocc:], with_t2=True)
        assert hr[0] == full[0] and hr[0].e_corr_ss == full[0].e_corr_ss and np.array_equal(hr[1], full[1])
    finally:
        hd.reset()
    t = dfmp2.times(d)
    assert t['total'] > 0, t


def _benzene(libpath, nocc_act):
    """benzene/cc-pVDZ (nvir = 93: diagonal and off-diagonal tile pairs, edge tiles) with random orthonormal orbitals and
    synthetic energies; the nocc_act highest occupied orbitals are active."""
    mol = gto.M(atom=geometry('benzene'), basis='cc-pvdz')
    d = DF(mol, 'cc-pvdz-jkfit', libpath=libpath).build()
    nao, nocc = d.nao, mol.nelectron // 2
    rng = np.random.RandomState(5)
    c = np.linalg.qr(rng.standard_normal((nao, nao)))[0]
    e = np.r_[np.sort(-1.0 - rng.random_sample(nocc)), np.sort(0.2 + rng.random_sample(nao - nocc))]
    assert nao - nocc == 93
    return d, d._cderi, c[:, nocc - nocc_act:nocc], c[:, nocc:], e[nocc - nocc_act:nocc], e[nocc:]


def _pair_screened_and_cart(libpath):
    """A pair-screened tensor (dropped columns read back as exact zeros) and a Cartesian molecule, against the model on the
    tensor read back."""
    atom = H2O + '; O 5 0 0; H 5 -0.757 0.587; H 5 0.757 0.587'
    mol = gto.M(atom=atom, basis='cc-pvdz')
    d = DF(mol, 'weigend', libpath=libpath, pair_tol=1e-8).build()
    assert d.pair_stats()[0] < d.pair_stats()[1]
    rng = np.random.RandomState(9)
    c = np.linalg.qr(rng.standard_normal((d.nao, d.nao)))[0]
    e = np.r_[np.sort(-1.0 - rng.random_sample(10)), np.sort(0.2 + rng.random_sample(d.nao - 10))]
    _check_r(d, d._cderi, c[:, 6:10], c[:, 10:40], e[6:10], e[10:40])
    mol = gto.M(atom=H2O, basis='cc-pvdz', cart=True)
    d = DF(mol, 'cc-pvdz-jkfit', libpath=libpath).build()
    assert d.nao == 25
    c = np.linalg.qr(rng.standard_normal((25, 25)))[0]
    e = np.r_[np.sort(-1.0 - rng.random_sample(5)), np.sort(0.2 + rng.random_sample(20))]
    _check_r(d, d._cderi, c[:, :5], c[:, 5:], e[:5], e[5:])


class _StandIn:
    """DFRMP2 / DFUMP2's call order (pyscf/mp/mp2.py:614-652): kernel -> ao2mo(mo_coeff) -> init_amps(mo_energy, mo_coeff, eris,
    with_t2), with split_mo_coeff / split_mo_energy of the active orbitals (_mo_splitter) and max_memory in MB."""

    def __init__(self, with_df, mo_coeff, mo_energy, nocc, frozen=(), max_memory=4000):
        self.with_df, self.mo_coeff, self.mo_energy = with_df, mo_coeff, mo_energy
        self.nocc, self.frozen, self.max_memory = nocc, frozen, max_memory
        self.unrestricted = isinstance(mo_coeff, tuple)

    def _masks(self, s):
        n = (self.mo_coeff[s] if self.unrestricted else self.mo_coeff).shape[1]
        nocc = self.nocc[s] if self.unrestricted else self.nocc
        act = np.ones(n, dtype=bool)
        act[list(self.frozen)] = False
        occ = np.arange(n) < nocc
        return [occ & ~act, occ & act, ~occ & act, ~occ & ~act]

    def split_mo_coeff(self):
        if self.unrestricted:
            return [[self.mo_coeff[s][:, m] for m in self._masks(s)] for s in (0, 1)]
        return [self.mo_coeff[:, m] for m in self._masks(0)]

    def split_mo_energy(self):
        if self.unrestricted:
            return [[self.mo_energy[s][m] for m in self._masks(s)] for s in (0, 1)]
        return [self.mo_energy[m] for m in self._masks(0)]

    def ao2mo(self, mo_coeff=None, ovL=None, ovL_to_save=None):
        raise AssertionError('the reference route would copy the whole tensor to the host here')

    def init_amps(self, mo_energy=None, mo_coeff=None, eris=None, with_t2=True):
        raise AssertionError('the reference route would contract on the CPU here')

    def kernel(self, with_t2=True):
        eris = self.ao2mo(self.mo_coeff)
        self.e_corr, self.t2 = self.init_amps(self.mo_energy, self.mo_coeff, eris, with_t2)
        self.e_corr_ss = getattr(self.e_corr, 'e_corr_ss', 0)
        self.e_corr_os = getattr(self.e_corr, 'e_corr_os', 0)
        self.e_corr = float(self.e_corr)
        return self.e_corr, self.t2


def _route(libpath):
    mol, e, c, d, B = _h2o_df(libpath)
    nocc = mol.nelectron // 2
    pt = dfmp2.patch(_StandIn(d, c, e, nocc, frozen=(0, 1, 5)))
    ec, t2 = pt.kernel()
    co, cv, eo, ev = _split(c, e, nocc, (0, 1, 5))
    e_ss, e_os, t2m = model_rmp2(B, d.nao, co, cv, eo, ev)
    assert type(ec) is float and abs(pt.e_corr_ss - e_ss) <= 1e-10 and abs(pt.e_corr_os - e_os) <= 1e-10
    assert t2.shape == (3, 3, 18, 18) and abs(t2 - t2m).max() <= 1e-12 * abs(t2m).max()
    eris = pt.ao2mo()
    assert (eris.nocc, eris.nvir, eris.naux) == (3, 18, d.get_naoaux())
    with pytest.raises(NotImplementedError, match='ovL'):
        pt.ao2mo(ovL=np.zeros(3))
    with pytest.raises(NotImplementedError, match='ovL'):
        pt.ao2mo(ovL_to_save='ovL.h5')
    small = dfmp2.patch(_StandIn(d, c, e, nocc, max_memory=0.01))
    with pytest.raises(MemoryError, match='with_t2 = False'):
        small.kernel()
    assert small.kernel(with_t2=False)[1] is None
    # DFUMP2
    pu = dfmp2.patch(_StandIn(d, (c, c), (e, e), (nocc, nocc - 1), frozen=(0,)))
    eu, t2u = pu.kernel()
    sp = [_split(c, e, n, (0,)) for n in (nocc, nocc - 1)]
    e_ss, e_os, t2m = model_ump2(B, d.nao, [s[0] for s in sp], [s[1] for s in sp], [s[2] for s in sp], [s[3] for s in sp])
    assert abs(pu.e_corr_ss - e_ss) <= 1e-10 and abs(pu.e_corr_os - e_os) <= 1e-10
    assert [x.shape for x in t2u] == [(4, 4, 19, 19), (4, 3, 19, 20), (3, 3, 20, 20)]


def _refusals(libpath):
    mol, e, c, d, B = _h2o_df(libpath)
    co, cv, eo, ev = c[:, :5], c[:, 5:], e[:5], e[5:]
    with pytest.raises(NotImplementedError, match='sharded'):
        dfmp2.kernel(DF(mol, _ri_basis(), libpath=libpath, shard=(0, 2)), co, cv, eo, ev)
    with pytest.raises(NotImplementedError, match='complex'):
        dfmp2.kernel(d, co + 0j, cv, eo, ev)
    with pytest.raises(NotImplementedError, match='complex'):
        dfmp2.ukernel(d, [co, co], [cv, cv + 0j], [eo, eo], [ev, ev])
    with pytest.raises(ValueError, match='nao'):
        dfmp2.kernel(d, co[1:], cv[1:], eo, ev)
    with pytest.raises(ValueError, match='nao'):
        dfmp2.ukernel(d, [co, co], [cv, cv[:-1]], [eo, eo], [ev, ev])
    with pytest.raises(ValueError, match='energies'):
        dfmp2.kernel(d, co, cv, eo[:-1], ev)


def test_h2o_cases_emulated(emu_lib):
    _h2o_cases(emu_lib)


def test_benzene_emulated(emu_lib):
    """Three active occupied orbitals against 93 virtual ones: tile pairs (0,0), (0,1), (1,1), the second tile an edge tile."""
    d, B, co, cv, eo, ev = _benzene(emu_lib, 3)
    _check_r(d, B, co, cv, eo, ev)
    _check_u(d, B, [co, co[:, 1:]], [cv, cv[:, :70]], [eo, eo[1:]], [ev, ev[:70]])


def test_pair_screened_and_cartesian_emulated(emu_lib):
    _pair_screened_and_cart(emu_lib)


def test_route_emulated(emu_lib):
    _route(emu_lib)


def test_refused_inputs_emulated(emu_lib):
    _refusals(emu_lib)


# ---- GPU -------------------------------------------------------------------------------------------------------------------

@pytest.mark.gpu
def test_small_cases_gpu():
    """The emulated cases on sm_90a."""
    _h2o_cases(None)
    _pair_screened_and_cart(None)
    _route(None)
    _refusals(None)


@pytest.mark.gpu
def test_benzene_gpu():
    """benzene/cc-pVDZ with all 21 occupied orbitals, RMP2 and UMP2."""
    d, B, co, cv, eo, ev = _benzene(None, 21)
    try:
        _check_r(d, B, co, cv, eo, ev)
        _check_u(d, B, [co, co[:, 1:]], [cv, cv[:, :70]], [eo, eo[1:]], [ev, ev[:70]])
    finally:
        d.reset()


@pytest.mark.gpu
def test_c60_window_gpu():
    """C60/def2-SVP (nvir 660, naux 4500) with the 20 highest occupied orbitals active: e_corr against DF.ao2mo((co, cv, co, cv))
    and the energy summed on the host, to 1e-9 Eh."""
    mol = gto.M(atom=geometry('c60'), basis='def2-svp')
    d = DF(mol).build()
    try:
        nao, nocc = d.nao, mol.nelectron // 2
        rng = np.random.RandomState(17)
        c = np.linalg.qr(rng.standard_normal((nao, nao)))[0]
        e = np.r_[np.sort(-1.0 - rng.random_sample(nocc)), np.sort(0.2 + rng.random_sample(nao - nocc))]
        co, cv, eo, ev = c[:, nocc - 20:nocc], c[:, nocc:], e[nocc - 20:nocc], e[nocc:]
        got = dfmp2.kernel(d, co, cv, eo, ev)[0]
        t = dfmp2.times(d)
        nv = cv.shape[1]
        ovov = d.ao2mo((co, cv, co, cv))
        ed = ex = 0.0
        for i in range(20):
            g = ovov[i * nv:(i + 1) * nv].reshape(nv, 20, nv).transpose(1, 0, 2)     # g[j, a, b] = (ia|jb)
            tt = g / (eo[i] + eo[:, None, None] - ev[None, :, None] - ev[None, None, :])
            ed += np.einsum('jab,jab', tt, g)
            ex -= np.einsum('jab,jba', tt, g)
        assert abs(got.e_corr_os - ed) < 1e-9 and abs(got.e_corr_ss - (ed + ex)) < 1e-9, (got.e_corr_os - ed, got.e_corr_ss - ed - ex)
        print('C60/def2-SVP 20-orbital window: e_corr %.12f, %s' % (got, t))
    finally:
        d.reset()
