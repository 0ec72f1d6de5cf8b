"""Direct RPA on the GPU (pyscf_b200.rpa: b200jk_df_rpa, df_rpa.cuh) — the RPA / URPA kernels of pyscf/gw/rpa.py:43-145 and
pyscf/gw/urpa.py:41-72.

The model is a numpy restatement of rpa.kernel and make_dielectric_matrix on a tensor: per frequency of the scaled
Gauss-Legendre grid, Pi = sum_s L_s chi_s L_s^T with chi_s = 2 e_ov f_ov / (w^2 + e_ov^2), and log det(I - Pi) from slogdet.
It is pinned to the reference's own identities on H2O/cc-pVDZ HF orbitals and the oracle's cc-pVDZ-RI tensor: at nw = 40 the
quadrature equals the plasmon formula 1/2 (sum omega_n^+ - tr A) of the N^6 RPA eigenproblem (rpa.py:311-323) to 1e-8 Eh, for
RHF and for UHF H2O+, and URPA with alpha = beta equals RPA (urpa.py:157-163).  The kernel is checked against the model on the
tensor read back with DF.loop(): e_corr within 1e-10 Eh, per-frequency log det and trace within 1e-10, Pi element-wise within
1e-12 max|Pi|.  The CPU emulation runs the same CTA code (tile list, both spin segments in one K, edge tiles, the epilogue and
the diagonal sums) on a host model of the fragments; the GPU tier repeats the cases on sm_90a and adds C60/def2-SVP against
Sylvester's identity on DF.ao2mo's (ia|jb)."""
import numpy as np
import pytest
import scipy.linalg

from pyscf_b200 import gto, rpa
from pyscf_b200.df import DF
from pyscf_b200.gto.mole import geometry
from test_df_mp2 import H2O, _h2o_df, _h2o_scf, _ri_basis, _split, _uhf, _unpack


# ---- the model ----------------------------------------------------------------------------------------------------------------

def _L(B, nao, co, cv):
    """L[P, i nvir + a] = C_occ[:, i]^T B_P C_vir[:, a]."""
    return np.einsum('pmn,mi,na->pia', _unpack(B, nao), co, cv, optimize=True).reshape(len(B), -1)


def _ls(B, nao, cos, cvs):
    return [_L(B, nao, co, cv) if co.shape[1] and cv.shape[1] else None for co, cv in zip(cos, cvs)]


def model_diel(Ls, e_ovs, f_ovs, omega, naux):
    """make_dielectric_matrix (rpa.py:100-130, urpa.py:41-72)."""
    diel = np.zeros((naux, naux))
    for L, e, f in zip(Ls, e_ovs, f_ovs):
        if L is not None:
            chi0 = 2.0 * e * f / (omega ** 2 + e ** 2)
            diel += (L * chi0) @ L.T
    return diel


def model_terms(Ls, e_ovs, f_ovs, omegas, naux):
    """(log det(I - Pi(w)), tr Pi(w)) per frequency."""
    ld, tr = [], []
    for w in omegas:
        diel = model_diel(Ls, e_ovs, f_ovs, w, naux)
        sign, v = np.linalg.slogdet(np.eye(naux) - diel)
        assert sign > 0
        ld.append(v)
        tr.append(np.trace(diel))
    return np.array(ld), np.array(tr)


def model_ecorr(Ls, e_ovs, f_ovs, naux, nw=40, x0=0.5):
    """rpa.kernel (rpa.py:77-92) with log(det(.)) taken as slogdet."""
    freqs, wts = rpa.scaled_legendre_roots(nw, x0)
    ld, tr = model_terms(Ls, e_ovs, f_ovs, freqs, naux)
    e = 0.0
    for w, a, b in zip(wts, ld, tr):
        e += w / (2.0 * np.pi) * a
        e += w / (2.0 * np.pi) * b
    return e


def _e_ov(eo, ev):
    return (eo[:, None] - ev).ravel()


def plasmon(Ls, e_ovs, f):
    """rpa.py:311-323: 1/2 (sum of the positive eigenvalues of [[A, B], [-B, -A]] - tr A), A = -e_ov + f VtV, B = f VtV, with the
    spins stacked into V (f = 2 for RPA, 1 for spin-blocked URPA)."""
    V = np.hstack([L for L in Ls if L is not None])
    a = np.diag(-np.concatenate(e_ovs)) + f * V.T @ V
    b = f * V.T @ V
    ev = scipy.linalg.eig(np.block([[a, b], [-b, -a]]))[0].real
    return 0.5 * (np.sum(ev[ev > 0]) - np.trace(a))


# ---- the model against the reference's identities (CPU, oracle only) ----------------------------------------------------------

def _h2o_tensor():
    mol, e, c = _h2o_scf()
    from oracle import oracle as O
    from pyscf_b200.gto.mole import make_auxmol
    B, nao = O.cholesky_eri(mol, make_auxmol(mol, _ri_basis()))
    return mol, e, c, B, nao


def test_model_plasmon_rhf():
    """RHF H2O: the nw = 40 quadrature against the N^6 plasmon formula, 1e-8 Eh (measured ~1e-9); at nw = 60 ~1e-13."""
    mol, e, c, B, nao = _h2o_tensor()
    nocc = mol.nelectron // 2
    co, cv, eo, ev = _split(c, e, nocc, ())
    Ls = _ls(B, nao, [co], [cv])
    eov = _e_ov(eo, ev)
    ref = plasmon(Ls, [eov], 2.0)
    q40 = model_ecorr(Ls, [eov], [np.full(eov.size, 2.0)], len(B), nw=40)
    q60 = model_ecorr(Ls, [eov], [np.full(eov.size, 2.0)], len(B), nw=60)
    assert abs(q40 - ref) < 1e-8, (q40, ref)
    assert abs(q60 - ref) < 1e-11, (q60, ref)
    assert -0.3 < ref < -0.2, ref


def test_model_plasmon_uhf_and_alpha_equals_beta():
    """UHF H2O+ (5 alpha, 4 beta, f_ov = 1, spin-blocked A / B) against the plasmon formula; URPA with alpha = beta is RPA."""
    mol, e, c, B, nao = _h2o_tensor()
    nel = (5, 4)
    orbs = _uhf(mol, nel, c)
    sp = [_split(orbs[k][1], orbs[k][0], nel[k], ()) for k in (0, 1)]
    Ls = _ls(B, nao, [x[0] for x in sp], [x[1] for x in sp])
    eovs = [_e_ov(x[2], x[3]) for x in sp]
    fovs = [np.ones(x.size) for x in eovs]
    q = model_ecorr(Ls, eovs, fovs, len(B))
    assert abs(q - plasmon(Ls, eovs, 1.0)) < 1e-8
    co, cv, eo, ev = _split(c, e, mol.nelectron // 2, ())
    Lr = _ls(B, nao, [co], [cv])
    eov = _e_ov(eo, ev)
    er = model_ecorr(Lr, [eov], [np.full(eov.size, 2.0)], len(B))
    eu = model_ecorr(Lr * 2, [eov] * 2, [np.ones(eov.size)] * 2, len(B))
    assert abs(er - eu) < 1e-12, (er, eu)


# ---- the kernel against the model (emulated, and on sm_90a) -----------------------------------------------------------------

def _check(d, B, cos, cvs, eovs, fovs, nw=40, diel_omega=0.7):
    """e_corr, per-frequency log det / trace and Pi(diel_omega) of the kernel against the model; returns the kernel's e_corr."""
    naux = len(B)
    Ls = _ls(B, d.nao, cos, cvs)
    got = rpa.kernel(d, cos, cvs, eovs, fovs, nw=nw)
    want = model_ecorr(Ls, eovs, fovs, naux, nw=nw)
    assert isinstance(got, float) and abs(got - want) <= 1e-10, (got, want, got - want)
    freqs = rpa.scaled_legendre_roots(nw)[0]
    ld, tr = rpa.kernel_terms(d, cos, cvs, eovs, fovs, freqs)
    mld, mtr = model_terms(Ls, eovs, fovs, freqs, naux)
    assert abs(ld - mld).max() <= 1e-10 and abs(tr - mtr).max() <= 1e-10, (abs(ld - mld).max(), abs(tr - mtr).max())
    pi = rpa.dielectric_matrix(d, cos, cvs, eovs, fovs, diel_omega)
    pm = model_diel(Ls, eovs, fovs, diel_omega, naux)
    assert pi.shape == (naux, naux) and np.array_equal(pi, pi.T)
    scale = max(abs(pm).max(), 1e-300)
    assert abs(pi - pm).max() <= 1e-12 * scale, abs(pi - pm).max() / scale
    return got


def _rhf_args(c, e, nocc, frozen=()):
    co, cv, eo, ev = _split(c, e, nocc, frozen)
    eov = _e_ov(eo, ev)
    return [co], [cv], [eov], [np.full(eov.size, 2.0)]


def _h2o_cases(libpath, bit_exact):
    """RPA with and without frozen orbitals, nocc = 1, a spin with no virtual orbitals, caller's f_ov, URPA of H2O+ with different
    alpha / beta sets and with alpha = beta; host rows and repeated calls."""
    mol, e, c, d, B = _h2o_df(libpath)
    nocc = mol.nelectron // 2
    full = _check(d, B, *_rhf_args(c, e, nocc))
    _check(d, B, *_rhf_args(c, e, nocc, (0, 1, 5)))
    _check(d, B, [c[:, 4:5]], [c[:, 5:]], [_e_ov(e[4:5], e[5:])], [np.full(19, 2.0)])            # nocc = 1
    # no virtual orbitals: Pi = 0, e_corr exactly 0
    assert rpa.kernel(d, c[:, :nocc], c[:, :0], np.zeros(0), np.zeros(0)) == 0.0
    assert not rpa.dielectric_matrix(d, c[:, :nocc], c[:, :0], np.zeros(0), np.zeros(0), 0.5).any()
    # f_ov of the caller's own (not 2), passed through unchanged
    cos, cvs, eovs, _ = _rhf_args(c, e, nocc)
    rng = np.random.RandomState(4)
    _check(d, B, cos, cvs, eovs, [1.0 + rng.random_sample(eovs[0].size)])
    # URPA: alpha = the RHF orbitals, beta = a rotated set with one electron fewer (the shape of H2O+), f_ov = 1
    rot = scipy.linalg.expm(0.05 * (lambda a: a - a.T)(rng.standard_normal((c.shape[1],) * 2)))
    cb, eb = c @ rot, e + 0.01 * rng.standard_normal(len(e))
    ucos, ucvs = [c[:, :nocc], cb[:, :nocc - 1]], [c[:, nocc:], cb[:, nocc - 1:]]
    ueovs = [_e_ov(e[:nocc], e[nocc:]), _e_ov(eb[:nocc - 1], eb[nocc - 1:])]
    ufovs = [np.ones(x.size) for x in ueovs]
    eu = _check(d, B, ucos, ucvs, ueovs, ufovs)
    # a spin with no virtual orbitals contributes nothing
    e1 = rpa.kernel(d, [c[:, :nocc], cb[:, :nocc]], [c[:, nocc:], cb[:, :0]], [ueovs[0], np.zeros(0)], [ufovs[0], np.zeros(0)])
    assert e1 == rpa.kernel(d, [c[:, :nocc]], [c[:, nocc:]], [ueovs[0]], [ufovs[0]])
    # URPA with alpha = beta and f_ov = 1 is RPA
    ea = rpa.kernel(d, [c[:, :nocc]] * 2, [c[:, nocc:]] * 2, [eovs[0]] * 2, [np.ones(eovs[0].size)] * 2)
    assert abs(ea - full) <= 1e-12, (ea, full)
    # repeated calls, and half of the rows on the host
    again = rpa.kernel(d, *_rhf_args(c, e, nocc))
    uagain = rpa.kernel(d, ucos, ucvs, ueovs, ufovs)
    naux = d.get_naoaux()
    hd = DF(mol, _ri_basis(), libpath=libpath).set_device_rows(naux // 2).build()
    try:
        assert hd.row_split() == (naux // 2, naux - naux // 2)
        hr = rpa.kernel(hd, *_rhf_args(c, e, nocc))
        hu = rpa.kernel(hd, ucos, ucvs, ueovs, ufovs)
    finally:
        hd.reset()
    same = (again, uagain, hr, hu) == (full, eu, full, eu)
    print('RPA H2O: repeated calls and host rows bit-identical: %s (differences %.1e %.1e %.1e %.1e)'
          % (same, again - full, uagain - eu, hr - full, hu - eu))
    if bit_exact:
        assert same
    else:
        assert max(abs(again - full), abs(uagain - eu), abs(hr - full), abs(hu - eu)) <= 1e-12
    t = rpa.times(d)
    assert t['total'] > 0 and set(t) == {'stage1', 'pi', 'factor', 'total'}, t


def _benzene(libpath, nocc_act):
    """benzene/cc-pVDZ with the cc-pVDZ-JKFIT tensor (naux not a multiple of 64: edge tiles), random orthonormal orbitals and
    synthetic energies; the nocc_act highest occupied orbitals are active."""
    mol = gto.M(atom=geometry('benzene'), basis='cc-pvdz')
    d = DF(mol, 'cc-pvdz-jkfit', libpath=libpath).build()
    nao, nocc = d.nao, mol.nelectron // 2
    assert d.get_naoaux() % 64 != 0
    rng = np.random.RandomState(5)
    c = np.linalg.qr(rng.standard_normal((nao, nao)))[0]
    e = np.r_[np.sort(-1.0 - rng.random_sample(nocc)), np.sort(0.2 + rng.random_sample(nao - nocc))]
    co, cv = c[:, nocc - nocc_act:nocc], c[:, nocc:]
    eov = _e_ov(e[nocc - nocc_act:nocc], e[nocc:])
    return d, d._cderi, co, cv, eov


def _pair_screened_and_cart(libpath):
    """A pair-screened tensor and a Cartesian molecule, against the model on the tensor read back."""
    mol = gto.M(atom=H2O + '; O 5 0 0; H 5 -0.757 0.587; H 5 0.757 0.587', basis='cc-pvdz')
    d = DF(mol, 'weigend', libpath=libpath, pair_tol=1e-8).build()
    assert d.pair_stats()[0] < d.pair_stats()[1]
    rng = np.random.RandomState(9)
    c = np.linalg.qr(rng.standard_normal((d.nao, d.nao)))[0]
    e = np.r_[np.sort(-1.0 - rng.random_sample(10)), np.sort(0.2 + rng.random_sample(d.nao - 10))]
    eov = _e_ov(e[6:10], e[10:40])
    _check(d, d._cderi, [c[:, 6:10]], [c[:, 10:40]], [eov], [np.full(eov.size, 2.0)], nw=8)
    mol = gto.M(atom=H2O, basis='cc-pvdz', cart=True)
    d = DF(mol, 'cc-pvdz-jkfit', libpath=libpath).build()
    assert d.nao == 25
    c = np.linalg.qr(rng.standard_normal((25, 25)))[0]
    e = np.r_[np.sort(-1.0 - rng.random_sample(5)), np.sort(0.2 + rng.random_sample(20))]
    eov = _e_ov(e[:5], e[5:])
    _check(d, d._cderi, [c[:, :5]], [c[:, 5:]], [eov], [np.full(eov.size, 2.0)], nw=8)


class _StandIn:
    """RPA / URPA's call order (rpa.py:188-227, urpa.py:75-107): kernel -> dump_flags -> ao2mo -> get_e_hf -> make_e_ov /
    make_f_ov -> make_dielectric_matrix per frequency -> e_hf, e_corr -> _finalize, with split_mo_coeff / split_mo_energy /
    split_mo_occ of the active orbitals (_mo_splitter)."""

    def __init__(self, with_df, mo_coeff, mo_energy, nocc, frozen=(), e_hf=-76.0):
        self.with_df, self.mo_coeff, self.mo_energy = with_df, mo_coeff, mo_energy
        self.nocc, self.frozen = nocc, frozen
        self.unrestricted = isinstance(mo_coeff, tuple)
        self._e_hf = e_hf
        self.e_hf = self.e_corr = None
        self.calls = []

    @property
    def e_tot(self):
        return self.e_hf + self.e_corr

    def _masks(self, s):
        n = (self.mo_coeff[s] if self.unrestricted else self.mo_coeff).shape[1]
        nocc = self.nocc[s] if self.unrestricted else self.nocc
        act = np.ones(n, dtype=bool)
        act[list(self.frozen)] = False
        occ = np.arange(n) < nocc
        return [occ & ~act, occ & act, ~occ & act, ~occ & ~act]

    def _split(self, x):
        if self.unrestricted:
            return [[x[s][m] if x[s].ndim == 1 else x[s][:, m] for m in self._masks(s)] for s in (0, 1)]
        return [x[m] if x.ndim == 1 else x[:, m] for m in self._masks(0)]

    def split_mo_coeff(self):
        return self._split(self.mo_coeff)

    def split_mo_energy(self):
        return self._split(self.mo_energy)

    def split_mo_occ(self):
        f = 1.0 if self.unrestricted else 2.0
        occ = tuple(f * (np.arange(len(e)) < n) for e, n in zip(self.mo_energy, self.nocc)) if self.unrestricted else \
            f * (np.arange(len(self.mo_energy)) < self.nocc)
        return self._split(occ)

    def dump_flags(self):
        self.calls.append('dump_flags')

    def get_e_hf(self):
        self.calls.append('get_e_hf')
        return self._e_hf

    def make_e_ov(self):
        if self.unrestricted:
            sp = self.split_mo_energy()
            return [(sp[s][1][:, None] - sp[s][2]).ravel() for s in (0, 1)]
        sp = self.split_mo_energy()
        return (sp[1][:, None] - sp[2]).ravel()

    def make_f_ov(self):
        if self.unrestricted:
            sp = self.split_mo_occ()
            return [(sp[s][1][:, None] - sp[s][2]).ravel() for s in (0, 1)]
        sp = self.split_mo_occ()
        return (sp[1][:, None] - sp[2]).ravel()

    def ao2mo(self, mo_coeff=None, ovL=None, ovL_to_save=None):
        raise AssertionError('the reference route would copy the whole tensor to the host here')

    def make_dielectric_matrix(self, omega, e_ov=None, f_ov=None, eris=None, max_memory=None, blksize=None):
        raise AssertionError('the reference route would read eris.get_ov_blk and multiply on the CPU here')

    def kernel(self, eris=None, nw=40, x0=0.5):
        raise AssertionError('the reference route would run here')

    def _finalize(self):
        self.calls.append('_finalize')


def _route(libpath):
    mol, e, c, d, B = _h2o_df(libpath)
    nocc = mol.nelectron // 2
    r = rpa.patch(_StandIn(d, c, e, nocc, frozen=(0, 1, 5)))
    ec = r.kernel()
    want = model_ecorr(_ls(B, d.nao, *_rhf_args(c, e, nocc, (0, 1, 5))[:2]), *_rhf_args(c, e, nocc, (0, 1, 5))[2:], len(B))
    assert type(ec) is float and ec == r.e_corr and abs(ec - want) <= 1e-10, (ec, want)
    assert r.e_hf == -76.0 and r.e_tot == r.e_hf + r.e_corr
    assert r.calls == ['dump_flags', 'get_e_hf', '_finalize'], r.calls
    eris = r.ao2mo()
    assert (eris.nocc, eris.nvir, eris.naux) == (3, 18, d.get_naoaux())
    with pytest.raises(NotImplementedError, match='device'):
        eris.get_ov_blk(0, 4)
    with pytest.raises(NotImplementedError, match='device'):
        eris.get_occ_blk(0, 4)
    with pytest.raises(NotImplementedError, match='ovL'):
        r.ao2mo(ovL=np.zeros(3))
    pi = r.make_dielectric_matrix(0.3)
    cos, cvs, eovs, fovs = _rhf_args(c, e, nocc, (0, 1, 5))
    pm = model_diel(_ls(B, d.nao, cos, cvs), eovs, fovs, 0.3, len(B))
    assert abs(pi - pm).max() <= 1e-12 * abs(pm).max()
    # URPA: alpha = beta = the RHF orbitals with one beta electron fewer
    u = rpa.patch(_StandIn(d, (c, c), (e, e), (nocc, nocc - 1), frozen=(0,)))
    eu = u.kernel(nw=20)
    sp = [_split(c, e, n, (0,)) for n in (nocc, nocc - 1)]
    eovs = [_e_ov(x[2], x[3]) for x in sp]
    want = model_ecorr(_ls(B, d.nao, [x[0] for x in sp], [x[1] for x in sp]), eovs, [np.ones(x.size) for x in eovs], len(B), nw=20)
    assert abs(eu - want) <= 1e-10 and u.e_tot == u.e_hf + eu
    assert (u.ao2mo().nocc, u.ao2mo().nvir) == ((4, 3), (19, 20))
    # complex orbitals: the reference's NotImplementedError before anything runs
    z = rpa.patch(_StandIn(d, c + 0j, e, nocc))
    with pytest.raises(NotImplementedError):
        z.kernel()
    assert z.calls == []


def _refusals(libpath, emulated):
    mol, e, c, d, B = _h2o_df(libpath)
    cos, cvs, eovs, fovs = _rhf_args(c, e, 5)
    with pytest.raises(NotImplementedError, match='sharded'):
        rpa.kernel(DF(mol, _ri_basis(), libpath=libpath, shard=(0, 2)), cos, cvs, eovs, fovs)
    with pytest.raises(NotImplementedError, match='complex'):
        rpa.kernel(d, [cos[0] + 0j], cvs, eovs, fovs)
    with pytest.raises(ValueError, match='nao'):
        rpa.kernel(d, [cos[0][1:]], [cvs[0][1:]], eovs, fovs)
    with pytest.raises(ValueError, match='e_ov'):
        rpa.kernel(d, cos, cvs, [eovs[0][:-1]], fovs)
    with pytest.raises(TypeError, match='with_df'):
        rpa.patch(_StandIn(object(), c, e, 5))
    if emulated:
        # e_ov of the wrong sign: chi > 0 and I - Pi is not positive definite at the small frequencies
        with pytest.raises(RuntimeError, match=r'not positive definite at omega = '):
            rpa.kernel(d, cos, cvs, [np.full(eovs[0].size, 0.05)], fovs)


def test_h2o_cases_emulated(emu_lib):
    _h2o_cases(emu_lib, True)


def test_benzene_emulated(emu_lib):
    """Three active occupied orbitals against 93 virtual ones at nw = 4; RPA and URPA with a second, smaller spin."""
    d, B, co, cv, eov = _benzene(emu_lib, 3)
    _check(d, B, [co], [cv], [eov], [np.full(eov.size, 2.0)], nw=4)
    eovb = eov.reshape(3, 93)[1:, :70].ravel()
    _check(d, B, [co, co[:, 1:]], [cv, cv[:, :70]], [eov, eovb], [np.ones(eov.size), np.ones(eovb.size)], nw=4)


def test_pair_screened_and_cartesian_emulated(emu_lib):
    _pair_screened_and_cart(emu_lib)


def test_route_emulated(emu_lib):
    _route(emu_lib)


def test_refused_inputs_emulated(emu_lib):
    _refusals(emu_lib, True)


# ---- GPU -------------------------------------------------------------------------------------------------------------------

@pytest.mark.gpu
def test_small_cases_gpu():
    """The emulated cases on sm_90a; repeated calls and host rows within 1e-12 Eh (cuSOLVER's potrf promises no bits)."""
    _h2o_cases(None, False)
    _pair_screened_and_cart(None)
    _route(None)
    _refusals(None, False)


@pytest.mark.gpu
def test_benzene_gpu():
    """benzene/cc-pVDZ with all 21 occupied orbitals, RPA and URPA, nw = 40."""
    d, B, co, cv, eov = _benzene(None, 21)
    try:
        _check(d, B, [co], [cv], [eov], [np.full(eov.size, 2.0)])
        eovb = eov.reshape(21, 93)[1:, :70].ravel()
        _check(d, B, [co, co[:, 1:]], [cv, cv[:, :70]], [eov, eovb], [np.ones(eov.size), np.ones(eovb.size)])
    finally:
        d.reset()


@pytest.mark.gpu
def test_c60_window_gpu():
    """C60/def2-SVP (naux 4500) with the 8 highest occupied orbitals against all 660 virtual ones (nov 5280), nw = 8: log det and
    trace per frequency and e_corr against Sylvester's identity on G = DF.ao2mo's (ia|jb): log det(I - L chi L^T) =
    log det(I + |chi|^1/2 G |chi|^1/2), tr Pi = sum chi_ia G_ia,ia; 1e-9 Eh on e_corr."""
    mol = gto.M(atom=geometry('c60'), basis='def2-svp')
    d = DF(mol).build()
    try:
        nao, nocc = d.nao, mol.nelectron // 2
        rng = np.random.RandomState(17)
        c = np.linalg.qr(rng.standard_normal((nao, nao)))[0]
        e = np.r_[np.sort(-1.0 - rng.random_sample(nocc)), np.sort(0.2 + rng.random_sample(nao - nocc))]
        co, cv = c[:, nocc - 8:nocc], c[:, nocc:]
        eov = _e_ov(e[nocc - 8:nocc], e[nocc:])
        fov = np.full(eov.size, 2.0)
        got = rpa.kernel(d, co, cv, eov, fov, nw=8)
        t = rpa.times(d)
        freqs, wts = rpa.scaled_legendre_roots(8)
        ld, tr = rpa.kernel_terms(d, co, cv, eov, fov, freqs)
        G = d.ao2mo((co, cv, co, cv))
        want = 0.0
        for k, (w, wt) in enumerate(zip(freqs, wts)):
            chi = 2.0 * eov * fov / (w ** 2 + eov ** 2)
            s = np.sqrt(-chi)
            sign, mld = np.linalg.slogdet(np.eye(len(eov)) + s[:, None] * G * s[None, :])
            assert sign > 0
            mtr = np.dot(chi, np.diag(G))
            assert abs(ld[k] - mld) < 1e-9 and abs(tr[k] - mtr) < 1e-9, (k, ld[k] - mld, tr[k] - mtr)
            want += wt / (2 * np.pi) * mld
            want += wt / (2 * np.pi) * mtr
        assert abs(got - want) < 1e-9, (got, want, got - want)
        print('C60/def2-SVP nov 5280 nw 8: e_corr %.12f (|d| %.1e), %s' % (got, abs(got - want), t))
    finally:
        d.reset()
