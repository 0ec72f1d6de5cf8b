"""Density fitting for Cartesian AOs (mol.cart = True): a Cartesian tensor cderi[naux_cart, ncart(ncart+1)/2] in a Cartesian
auxiliary basis, as the reference builds it (make_auxmol copies mol.cart, pyscf/df/addons.py:245; cholesky_eri runs
int3c2e_cart / int2c2e_cart, pyscf/df/incore.py:144-149).  Checked against tests/cart_oracle.py (the oracle library's Cartesian
integral functions), which is itself pinned to the spherical oracle here.

Bars.  Cartesian auxiliary bases are much worse conditioned than spherical ones (their d/g shells carry r^2-type lower-l
components).  For H2O/cc-pVDZ with cc-pvdz-jkfit (metric condition number 2e10) and weigend (4e7), integral noise of 1e-15
relative moves J/K by <= 4e-13, so the usual bars hold: tensor 1e-10, J/K 1e-9.  He-Ne/cc-pVTZ with def2-universal-jkfit
(2.3e11, Cartesian g auxiliaries) moves K by up to 6.3e-10 under the same noise: J/K are compared at 1e-8 there, and its tensor
columns, which the same probe moves by up to HENE_COL_NOISE = 9.6e-8, at 10x that.
GPU: the same cases through the sm_90a build, and C60/cc-pVDZ (nao 900, naux 4860) against tests/golden/df_size_c60_cart.npz."""
import os
import subprocess
import sys

import numpy as np
import pytest

import cart_oracle as C
from pyscf_b200 import gto
from pyscf_b200.df import DF, TaggedDM, density_fit
from pyscf_b200.gto.mole import geometry, make_auxmol
from oracle import oracle as O

H2O = 'O 0 0 0; H 0 -0.757 0.587; H 0 0.757 0.587'
HENE = 'He 0 0 0; Ne 1.2 0.3 0'
# name: (atom, basis, auxbasis, J/K bar, tensor bar)
# max |d cderi| of the He-Ne tensor (|cderi| up to 2.3) over three draws of 1e-15 relative noise on (ij|P) and (P|Q): 1.9e-8 .. 9.6e-8
HENE_COL_NOISE = 9.6e-8
CASES = {'h2o_jkfit': (H2O, 'cc-pvdz', 'cc-pvdz-jkfit', 1e-9, 1e-10),
         'h2o_weigend': (H2O, 'cc-pvdz', 'weigend', 1e-9, 1e-10),
         'hene': (HENE, 'cc-pvtz', 'def2-universal-jkfit', 1e-8, 10 * HENE_COL_NOISE)}
_REF = {}


def _ref(name, omega=None):
    key = (name, omega)
    if key not in _REF:
        atom, basis, aux = CASES[name][:3]
        mol = gto.M(atom=atom, basis=basis, cart=True)
        _REF[key] = C.cholesky_eri(mol, make_auxmol(mol, aux), omega=omega)
    return _REF[key]


def _mol(name):
    atom, basis, aux = CASES[name][:3]
    return gto.M(atom=atom, basis=basis, cart=True), aux


def _set_kblock(d, kb):
    h = d._handle
    h.check(h.lib.b200jk_df_set_kblock(h._h, int(kb), -1), 'b200jk_df_set_kblock')


def _inputs(nao, seed=1):
    """Two orbital-tagged densities (one orbital set per density) and two general densities with hermi 0 and 1, n_dm = 2."""
    rng = np.random.RandomState(seed)
    c1, c2 = (np.linalg.qr(rng.standard_normal((nao, 4)))[0] * np.sqrt(2.0) for _ in range(2))
    dm_g = rng.random_sample((2, nao, nao))
    dm_s = dm_g + dm_g.transpose(0, 2, 1)
    dms_t = np.array([c1 @ c1.T, c2 @ c2.T])
    return {'tagged': (TaggedDM(dms_t, mo_coeff=np.array([c1, c2]), mo_occ=np.full((2, 4), 1.0)), 1, dms_t),
            'general0': (dm_g, 0, dm_g), 'general1': (dm_s, 1, dm_s)}


# ---- the Cartesian oracle itself -------------------------------------------------------------------------------------------

def test_cart_oracle_against_spherical_oracle():
    """Through the cart -> sph map T (identity on s/p, the oracle's c2s rows for l >= 2), the Cartesian integrals give the
    spherical oracle's: overlap, kinetic, nuclear attraction, (P|Q), (ij|P) and the Schwarz bounds of s/p-only shell pairs."""
    mol, aux = _mol('hene')
    sph = gto.M(atom=HENE, basis='cc-pvtz')
    T = C.cart2sph(mol)
    for kind in ('ovlp', 'kin'):
        assert abs(T.T @ C.int1e(mol, kind) @ T - O.int1e(sph, kind)).max() < 1e-12, kind
    assert abs(T.T @ C.nuc(mol) @ T - O.int1e(sph, 'nuc')).max() < 1e-12
    amol, asph = make_auxmol(mol, aux), make_auxmol(sph, aux)
    Ta = C.cart2sph(amol)
    assert abs(Ta.T @ C.int2c2e(amol) @ Ta - O.int2c2e(asph)).max() < 1e-12
    j3 = C.int3c2e(mol, amol)
    j3 = np.tensordot(np.tensordot(np.tensordot(j3, Ta, (2, 0)), T, (1, 0)), T, (0, 0)).transpose(2, 1, 0)
    assert abs(j3 - O.int3c2e(sph, asph)).max() < 1e-12
    qc, qs = C.q_cond(mol), O.q_cond(sph)
    low = mol._bas[:, 1] < 2
    assert abs(qc[np.ix_(low, low)] - qs[np.ix_(low, low)]).max() < 1e-13


# ---- tensor and J/K -------------------------------------------------------------------------------------------------------

def _check_tensor_jk(name, libpath, engines=('tcgen05', 'dgemm')):
    mol, aux = _mol(name)
    bar_jk, bar_col = CASES[name][3:]
    ref, nao = _ref(name)
    assert nao == mol.nao_nr(cart=True) and nao > mol.nao_nr(cart=False)
    d = DF(mol, aux, libpath=libpath).build()
    assert d.nao == nao and d.get_naoaux() == ref.shape[0] == make_auxmol(mol, aux).nao_nr(cart=True)
    assert abs(d._cderi - ref).max() < bar_col, abs(d._cderi - ref).max()
    for eng in engines:
        d.set_k_engine(eng, 7)
        for kind, (dm, hermi, dms) in _inputs(nao).items():
            vj, vk = d.get_jk(dm, hermi=hermi)
            rj, rk = O.df_get_jk(ref, nao, dms)
            assert abs(vj - rj).max() < bar_jk and abs(vk - rk).max() < bar_jk, (eng, kind, abs(vj - rj).max(), abs(vk - rk).max())
    d.reset()


@pytest.mark.parametrize('name', list(CASES))
def test_tensor_jk_emulated(emu_lib, name):
    """Tensor against the Cartesian oracle, naux = the Cartesian auxiliary count, J/K of tagged and general densities (hermi 0
    and 1, n_dm = 2) with both K engines."""
    _check_tensor_jk(name, emu_lib)


def test_direct_j_and_range_separation_emulated(emu_lib):
    """The integral-direct J (no tensor) equals the tensor's J; a range_coulomb(-0.3) child matches the oracle with omega.  The
    erf(0.3) metric of the Cartesian auxiliary basis is not positive definite (smallest eigenvalue ~ -1e-14): it takes the
    eigendecomposition fallback, which only the GPU build has, so +0.3 runs in the GPU test."""
    _check_direct_rsh(emu_lib, (-0.3,))


def _check_direct_rsh(libpath, omegas):
    mol, aux = _mol('h2o_weigend')
    ref, nao = _ref('h2o_weigend')
    dms = _inputs(nao)['general1'][2]
    dj = DF(mol, aux, libpath=libpath)
    vj_direct = dj.get_jk(dms, hermi=1, with_k=False)[0]
    assert dj._handle is None                   # served by the integral-direct path
    vj_t = DF(mol, aux, libpath=libpath).build().get_jk(dms, hermi=1)[0]
    assert abs(vj_direct - vj_t).max() < 1e-10
    d = DF(mol, aux, libpath=libpath).build()
    for omega in omegas:
        rref, _ = _ref('h2o_weigend', omega)
        child = d.range_coulomb(omega)
        assert child.nao == nao
        vj, vk = d.get_jk(dms, hermi=1, omega=omega)
        rj, rk = O.df_get_jk(rref, nao, dms)
        assert abs(vj - rj).max() < 1e-9 and abs(vk - rk).max() < 1e-9, omega


def test_pair_screening_emulated(emu_lib):
    """Two Cartesian H2O 5 A apart: the kept columns are the Cartesian oracle's q_cond >= tol (per segment of a general
    contraction) and J/K stay inside the bounds of DESIGN.md §3."""
    import test_df_pairscreen as PS
    atom = H2O + '; O 5 0 0; H 5 -0.757 0.587; H 5 0.757 0.587'
    mol, tol = gto.M(atom=atom, basis='cc-pvdz', cart=True), 1e-8
    ref, nao = C.cholesky_eri(mol, make_auxmol(mol, 'weigend'))
    seg = PS._segmented(mol)
    assert seg.cart and seg.nbas > mol.nbas
    q = PS._ao_q(seg, C.q_cond(seg))
    d = DF(mol, 'weigend', libpath=emu_lib, pair_tol=tol).build()
    ncol, npair = d.pair_stats()
    assert npair == nao * (nao + 1) // 2 and 0.3 < ncol / npair < 0.9, (ncol, npair)
    _, kept = PS._kept_mask(d, nao)
    qp = PS._tril(q)
    near = abs(qp / tol - 1.0) < 1e-9
    assert np.array_equal(kept[~near], (qp >= tol)[~near])
    assert (np.linalg.norm(ref, axis=0)[~kept] < tol).all()
    for kind, (dm, hermi, dms) in _inputs(nao).items():
        vj, vk = d.get_jk(dm, hermi=hermi)
        rj, rk = O.df_get_jk(ref, nao, dms)
        bj, bk = PS._bounds(ref, q, kept, dms)
        assert (abs(vj - rj) <= bj * (1 + 1e-6) + 1e-9).all(), kind
        assert (abs(vk - rk) <= bk * (1 + 1e-6) + 1e-9).all(), kind


def test_host_rows_and_shards_emulated(emu_lib):
    """Forced host rows (0 and naux/3 on the device) and two shard ranks summed give the resident handle's J/K to 1e-12."""
    mol, aux = _mol('h2o_jkfit')
    nao = mol.nao
    d0 = DF(mol, aux, libpath=emu_lib).build()
    naux = d0.get_naoaux()
    inputs = _inputs(nao)
    want = {k: d0.get_jk(v[0], hermi=v[1]) for k, v in inputs.items()}
    for cap in (0, naux // 3):
        d = DF(mol, aux, libpath=emu_lib).set_device_rows(cap).build()
        assert d.row_split() == (cap, naux - cap)
        _set_kblock(d, max(1, (naux - cap) // 5))
        for kind, (dm, hermi, _) in inputs.items():
            vj, vk = d.get_jk(dm, hermi=hermi)
            assert abs(vj - want[kind][0]).max() < 1e-12 and abs(vk - want[kind][1]).max() < 1e-12, (cap, kind)
    dm = inputs['general0'][0]
    vj, vk = np.zeros_like(want['general0'][0]), np.zeros_like(want['general0'][1])
    for rank in range(2):
        pj, pk = DF(mol, aux, libpath=emu_lib, shard=(rank, 2)).build().get_jk(dm, hermi=0)
        vj += pj
        vk += pk
    assert abs(vj - want['general0'][0]).max() < 1e-12 and abs(vk - want['general0'][1]).max() < 1e-12


def test_interchange_emulated(emu_lib, tmp_path):
    """loop(), cderi_columns(), save() and an assigned _cderi use the Cartesian layout [naux_cart, ncart(ncart+1)/2]; a tensor
    of the spherical layout is refused for a Cartesian molecule."""
    mol, aux = _mol('h2o_weigend')
    ref, nao = _ref('h2o_weigend')
    npair = nao * (nao + 1) // 2
    d = DF(mol, aux, libpath=emu_lib).build()
    full = np.vstack(list(d.loop(blksize=7)))
    assert full.shape == (ref.shape[0], npair) and abs(full - ref).max() < 1e-10
    cols = np.array([0, 1, 5, 17, npair - 1])
    assert np.array_equal(d.cderi_columns(cols), full[:, cols])
    path = d.save(str(tmp_path / 'cart.npy'))
    assert np.array_equal(np.load(path), full)
    d2 = DF(mol, aux, libpath=emu_lib)
    d2._cderi = path
    dm = _inputs(nao)['general1'][0]
    a, b = d.get_jk(dm, hermi=1), d2.get_jk(dm, hermi=1)
    assert abs(a[0] - b[0]).max() < 1e-12 and abs(a[1] - b[1]).max() < 1e-12
    assert np.array_equal(d2._cderi, full)
    nsph = mol.nao_nr(cart=False)
    d3 = DF(mol, aux, libpath=emu_lib)
    d3._cderi = np.zeros((3, nsph * (nsph + 1) // 2))
    with pytest.raises(RuntimeError, match='cderi must have shape'):
        d3.build()


def test_mixed_bases_raise(emu_lib):
    """Cartesian orbitals with a spherical auxmol, or the reverse, fail with the reference's messages
    (pyscf/df/incore.py:144-147); only a user-assigned auxmol can mix them."""
    mol, aux = _mol('h2o_weigend')
    sph = gto.M(atom=H2O, basis='cc-pvdz')
    d = DF(mol, aux, libpath=emu_lib)
    d.auxmol = make_auxmol(sph, aux)
    with pytest.raises(RuntimeError, match='Cartesian orbitals for mol and spherical orbitals for auxmol not supported'):
        d.build()
    with pytest.raises(RuntimeError, match='Cartesian orbitals for mol'):
        d.get_jk(np.eye(mol.nao), with_k=False)
    d = DF(sph, aux, libpath=emu_lib)
    d.auxmol = make_auxmol(mol, aux)
    with pytest.raises(NotImplementedError, match='int3c2e_ssc'):
        d.build()


def test_density_fit_routes_to_cartesian_df(emu_lib):
    """density_fit on a Cartesian mean-field object gives a with_df whose J/K run over the Cartesian AOs."""

    class StandInSCF:
        def __init__(self, mol):
            self.mol = mol

        def get_jk(self, mol=None, dm=None, hermi=1, with_j=True, with_k=True, omega=None):
            raise AssertionError('the exact path is not taken')

    mol, aux = _mol('h2o_weigend')
    ref, nao = _ref('h2o_weigend')
    dfmf = density_fit(StandInSCF(mol), auxbasis=aux)
    dfmf.with_df._libpath = emu_lib
    dm = _inputs(nao)['general1'][0]
    vj, vk = dfmf.get_jk(mol, dm)
    assert dfmf.with_df.nao == nao == vj.shape[-1]
    rj, rk = O.df_get_jk(ref, nao, dm)
    assert abs(vj - rj).max() < 1e-9 and abs(vk - rk).max() < 1e-9


# ---- SCF energies ---------------------------------------------------------------------------------------------------------

def _scf(libpath, use_df):
    from pyscf_b200.jk import VHFOpt
    from pyscf_b200.scf import RHF
    mol = gto.M(atom=H2O, basis='cc-pvdz', cart=True)
    s = C.int1e(mol, 'ovlp')
    h = C.int1e(mol, 'kin') + C.nuc(mol)
    if use_df:
        eng = DF(mol, 'weigend', libpath=libpath).build()

        def get_jk(dm, co):
            return eng.get_jk(TaggedDM(dm, mo_coeff=co, mo_occ=np.full(co.shape[1], 2.0)))
    else:
        eng = VHFOpt(mol, libpath=libpath)

        def get_jk(dm, co):
            return eng.get_jk(dm, hermi=1)
    mf = RHF(mol, get_jk, h, s)
    return mf.kernel(), mf.converged


# pyscf/df/test/test_df_jk.py:66-70 (DF-UHF of closed-shell H2O, which converges to the RHF solution) and
# pyscf/scf/test/test_rhf.py:418-422
E_DF_CART, E_CART = -76.026760700636046, -76.027107008870573


def test_scf_energies_emulated(emu_lib):
    e, ok = _scf(emu_lib, True)
    assert ok and abs(e - E_DF_CART) < 1e-8, e
    e, ok = _scf(emu_lib, False)
    assert ok and abs(e - E_CART) < 1e-8, e


# ---- GPU ------------------------------------------------------------------------------------------------------------------

@pytest.mark.gpu
@pytest.mark.parametrize('name', list(CASES))
def test_tensor_jk_gpu(name):
    _check_tensor_jk(name, None)


@pytest.mark.gpu
def test_direct_j_and_range_separation_gpu():
    _check_direct_rsh(None, (0.3, -0.3))


@pytest.mark.gpu
def test_scf_energies_gpu():
    e, ok = _scf(None, True)
    assert ok and abs(e - E_DF_CART) < 1e-8, e
    e, ok = _scf(None, False)
    assert ok and abs(e - E_CART) < 1e-8, e


def _c60_bar(z, key=('noise_dj', 'noise_dk')):
    """1e-9 when 1e-15 relative integral noise moves the fixture's values by less than 1e-10, else 10x that spread (the probe of
    tools/make_golden_df_size.py).  C60/cc-pVDZ Cartesian, metric condition number 7.1e10: J/K move by 7.6e-12 / 2.1e-11, so their
    bar is 1e-9; the sampled tensor columns move by 3.0e-10, so theirs is 3.0e-9."""
    spread = max(float(z[k]) for k in key)
    return 1e-9 if spread < 1e-10 else 10 * spread


def _c60_cart(cap=-1, pair_tol=None):
    import df_size_check as S
    z = S.load('c60_cart')
    assert z is not None, 'fixture missing: python tools/make_golden_df_size.py c60_cart'
    mol = gto.M(atom=geometry('c60'), basis='cc-pvdz', cart=True)
    return S, z, mol, DF(mol, 'cc-pvdz-jkfit', pair_tol=pair_tol).set_device_rows(cap).build()


def _c60_check(S, z, d, mol):
    """Fixture columns and slab J/K with both K engines within the bar, and int8 against DGEMM on the SCF-like density."""
    bar = _c60_bar(z)
    assert d.nao == mol.nao == int(z['nao']) == 900 and d.get_naoaux() == int(z['naux']) == 4860
    dc = S.check_columns(d, z)
    c = S.slab_coeff(z)
    occ = np.full(c.shape[1], 2.0)
    dm = 2.0 * c.dot(c.T)
    out = {}
    for eng in ('tcgen05', 'dgemm'):
        d.set_k_engine(eng, 7)
        vj1, vk1 = d.get_jk(TaggedDM(dm, mo_coeff=c, mo_occ=occ), hermi=1)
        r1 = S.compare_jk(z, vj1, vk1)
        vj2, vk2 = d.get_jk(dm, hermi=1)
        r2 = S.compare_jk(z, vj2, vk2)
        for r in (r1, r2):
            assert max(r['max_abs_dJ'], r['max_abs_dK'], r['max_abs_dK_diag']) < bar, (eng, r, bar)
        out[eng] = (vj1, vk1, vj2, vk2)
    rng = np.random.RandomState(1)
    co, _ = np.linalg.qr(rng.standard_normal((mol.nao, int(z['nocc']))))
    dms = 2.0 * co.dot(co.T)
    tag = TaggedDM(dms, mo_coeff=co, mo_occ=np.full(co.shape[1], 2.0))
    d.set_k_engine('tcgen05', 7)
    vk3 = d.get_jk(tag, hermi=1, with_j=False)[1]
    d.set_k_engine('dgemm', 7)
    vk4 = d.get_jk(tag, hermi=1, with_j=False)[1]
    d.set_k_engine('tcgen05', 7)
    eng_dev = float(abs(vk3 - vk4).max())
    assert eng_dev < bar, eng_dev
    bar_col = _c60_bar(z, ('noise_dcol',))
    print('c60 cart: cond %.2e, noise spread J %.1e K %.1e cols %.1e, bars %.1e / %.1e | cols %.1e | tagged %s | general %s | '
          'int8 vs dgemm %.1e' % (float(z['cond']), float(z['noise_dj']), float(z['noise_dk']), float(z['noise_dcol']), bar, bar_col,
                                  dc, r1, r2, eng_dev))
    assert dc < bar_col, dc
    return out


_C60 = {}


def _c60_resident():
    if not _C60:
        S, z, mol, d = _c60_cart()
        try:
            assert d.row_split()[1] == 0
            _C60['naux'] = d.get_naoaux()
            _C60['out'] = _c60_check(S, z, d, mol)
        finally:
            d.reset()
    return _C60['out']


@pytest.mark.gpu
def test_c60_cart_fixture_gpu():
    """C60/cc-pVDZ Cartesian (15.8 GB tensor) against the size fixture with both K engines."""
    _c60_resident()


@pytest.mark.gpu
@pytest.mark.parametrize('variant', ['half_host', 'pair_tol_1e-300'])
def test_c60_cart_variants_gpu(variant):
    """Half of the rows in host memory, and pair screening that keeps every column with a surviving primitive pair, against the
    fixture and within 1e-10 of the resident dense build."""
    want = _c60_resident()
    if variant == 'half_host':
        S, z, mol, d = _c60_cart(cap=_C60['naux'] // 2)
    else:
        S, z, mol, d = _c60_cart(pair_tol=1e-300)
    try:
        got = _c60_check(S, z, d, mol)
        for eng in got:
            for a, b in zip(got[eng], want[eng]):
                assert abs(a - b).max() < 1e-10, (variant, eng, abs(a - b).max())
    finally:
        d.reset()


def _c60_unfused():
    S, z, mol, d = _c60_cart()
    try:
        _c60_check(S, z, d, mol)
    finally:
        d.reset()


@pytest.mark.gpu
def test_c60_cart_unfused_y_gpu():
    """The C60 Cartesian check with B200JK_NO_YFUSE=1, in a fresh process because the variable is read once per process."""
    here = os.path.dirname(os.path.abspath(__file__))
    code = 'import sys; sys.path[:0] = [%r, %r]; import test_df_cart as T; T._c60_unfused()' % (here, os.path.dirname(here))
    r = subprocess.run([sys.executable, '-c', code], env=dict(os.environ, B200JK_NO_YFUSE='1'), capture_output=True, text=True,
                       timeout=1800)
    assert r.returncode == 0, r.stdout[-2000:] + r.stderr[-4000:]
