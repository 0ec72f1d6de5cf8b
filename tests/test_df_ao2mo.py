"""MO and AO integrals from the density-fitting tensor: DF.ao2mo = get_mo_eri and DF.get_eri = get_ao_eri (pyscf/df/df.py:269-296),
the entry points of MP2, DF-CASSCF and DF-NEVPT2 on a fitted SCF (b200jk_df_ao2mo / b200jk_df_get_ao_eri, df_ao2mo.cuh).

Every case is checked twice: against a float64 numpy transform of the same tensor read back with DF.loop(), element by element
within 1e-12 ||L_ij|| ||L_kl|| (norms over the auxiliary index, the Cauchy-Schwarz scale of the element), and against the same
transform of the oracle's tensor (oracle.cholesky_eri, or the Cartesian oracle) within 1e-9.  The CPU emulation runs the same
GEMM tiling, packed-row loader, s2 packing and band pipeline on a host model of the 8x8x4 FP64 fragments; the GPU tier repeats
the small cases on sm_90a and adds benzene/cc-pVTZ ovov and a 16-orbital active space of C60/def2-SVP."""
import numpy as np
import pytest

from pyscf_b200 import gto
from pyscf_b200.df import DF, TaggedDM
from pyscf_b200.gto.mole import geometry, make_auxmol
from pyscf_b200.scf import RHF
from oracle import oracle as O

H2O = 'O 0 0 0; H 0 -0.757 0.587; H 0 0.757 0.587'
AUX = 'cc-pvdz-jkfit'


def _unpack(B, nao):
    """[nrow, npair] packed rows -> [nrow, nao, nao]."""
    out = np.zeros((len(B), nao, nao))
    i, j = np.tril_indices(nao)
    out[:, i, j] = B
    out[:, j, i] = B
    return out


def _half(Bf, c1, c2, s2):
    """L[P, ij] of one pair: s2 rows i(i+1)/2 + j (i >= j), else i n2 + j."""
    L = np.einsum('pmn,mi,nj->pij', Bf, c1, c2, optimize=True)
    if s2:
        i, j = np.tril_indices(c1.shape[1])
        return L[:, i, j]
    return L.reshape(len(Bf), -1)


def _np_ao2mo(B, nao, cs, s12, s34):
    """out, ||L_ij||, ||L_kl||."""
    Bf = _unpack(B, nao)
    L1 = _half(Bf, cs[0], cs[1], s12)
    L2 = _half(Bf, cs[2], cs[3], s34)
    return L1.T @ L2, np.linalg.norm(L1, axis=0), np.linalg.norm(L2, axis=0)


def _check(got, B, ref, nao, cs, s12, s34):
    want, n1, n2 = _np_ao2mo(B, nao, cs, s12, s34)
    assert got.shape == want.shape and got.dtype == np.float64, (got.shape, want.shape)
    bar = 1e-12 * np.outer(n1, n2)
    err = abs(got - want)
    assert (err <= bar).all(), (err - bar).max()
    want2 = _np_ao2mo(ref, nao, cs, s12, s34)[0]
    assert abs(got - want2).max() < 1e-9, abs(got - want2).max()


def _set_tile(d, rows):
    h = d._handle
    h.check(h.lib.b200jk_df_set_ao2mo_tile(h._h, int(rows)), 'b200jk_df_set_ao2mo_tile')


_CACHE = {}


def _h2o(libpath):
    """H2O/cc-pVDZ + cc-pvdz-jkfit: the DF object, the read-back tensor, the oracle's tensor and converged RHF orbitals."""
    if libpath not in _CACHE:
        mol = gto.M(atom=H2O, basis='cc-pvdz')
        d = DF(mol, AUX, libpath=libpath).build()
        ref, nao = O.cholesky_eri(mol, make_auxmol(mol, AUX))
        s = O.int1e(mol, 'ovlp')
        hcore = O.int1e(mol, 'kin') + O.int1e(mol, 'nuc')
        mf = RHF(mol, lambda dm, co: d.get_jk(TaggedDM(dm, mo_coeff=co, mo_occ=np.full(co.shape[1], 2.0))), hcore, s)
        mf.kernel()
        assert mf.converged
        _CACHE[libpath] = (mol, d, d._cderi, ref, nao, mf)
    return _CACHE[libpath]


def _orbital_cases(mo, nocc):
    """(name, mo_coeffs, compact, s12, s34) of the cases a post-SCF code hands to ao2mo."""
    nao, nmo = mo.shape
    co, cv = mo[:, :nocc], mo[:, nocc:]
    cas = mo[:, 2:8]
    rng = np.random.RandomState(7)
    d1, d2, d3, d4 = (rng.standard_normal((nao, n)) for n in (3, 5, 4, 2))
    return [('mo_compact', mo, True, True, True),
            ('mo_s1', mo, False, False, False),
            ('ovov', (co, cv, co, cv), True, False, False),
            ('mp_mp', [mo, cas, mo, cas], False, False, False),                  # pyscf/mrpt/dfnevpt2.py:196-199
            ('paaa', [mo, cas, cas, cas], False, False, False),                  # pyscf/mcscf/df.py:140
            ('aaaa', cas, True, True, True),                                     # mcscf/casci.py:373
            ('distinct', (d1, d2, d3, d4), True, False, False),
            ('fortran', (np.asfortranarray(co), cv, np.asfortranarray(cas), cas), True, False, True),
            ('strided', (mo[:, ::2], mo[:, 1::3], mo[:, ::2], mo[:, ::2]), True, False, True),
            ('single', mo[:, :1], True, True, True),
            ('single_s1', (mo[:, 3:4], mo[:, 5:6], mo[:, 3:4], mo[:, :nmo]), True, False, False)]


def _run_orbital_cases(d, B, ref, nao, mo, nocc):
    for name, cs, compact, s12, s34 in _orbital_cases(mo, nocc):
        four = (cs,) * 4 if isinstance(cs, np.ndarray) else cs
        got = d.ao2mo(cs, compact=compact)
        n = [c.shape[1] for c in four]
        assert got.shape == (n[0] * (n[0] + 1) // 2 if s12 else n[0] * n[1], n[2] * (n[2] + 1) // 2 if s34 else n[2] * n[3]), name
        _check(got, B, ref, nao, [np.asarray(c) for c in four], s12, s34)


def _mp2_energy(eri_ovov, mo_energy, nocc):
    """RMP2 correlation energy from (ia|jb) reshaped as mp2.py:808-830 does it."""
    nvir = len(mo_energy) - nocc
    eia = mo_energy[:nocc, None] - mo_energy[None, nocc:]
    e = 0.0
    for i in range(nocc):
        gi = eri_ovov[i * nvir:(i + 1) * nvir].reshape(nvir, nocc, nvir).transpose(1, 0, 2)
        t2i = gi.conj() / (eia[:, :, None] + eia[i][None, None, :])
        e += np.einsum('jab,jab', t2i, gi) * 2 - np.einsum('jab,jba', t2i, gi)
    return e


# ---- CPU emulation ---------------------------------------------------------------------------------------------------------

def test_orbital_cases_emulated(emu_lib):
    """2-D coefficients (compact on / off), ovov, the CASSCF / NEVPT2 shapes, four distinct sets, Fortran-ordered and strided
    inputs, single orbitals: against numpy on the read-back tensor and on the oracle's tensor."""
    mol, d, B, ref, nao, mf = _h2o(emu_lib)
    _run_orbital_cases(d, B, ref, nao, mf.mo_coeff, mol.nelectron // 2)


def test_iden_coeffs_rule_emulated(emu_lib):
    """An equal copy is the same set (s2); a copy perturbed by 1e-12 is not (s1), as iden_coeffs decides."""
    mol, d, B, ref, nao, mf = _h2o(emu_lib)
    mo = mf.mo_coeff[:, :6]
    copy = mo.copy()
    bumped = mo + 1e-12
    got = d.ao2mo((mo, copy, mo, copy))
    assert got.shape == (21, 21)
    _check(got, B, ref, nao, [mo, copy, mo, copy], True, True)
    got = d.ao2mo((mo, bumped, mo, mo))
    assert got.shape == (36, 21)
    _check(got, B, ref, nao, [mo, bumped, mo, mo], False, True)
    assert d.get_mo_eri == d.ao2mo and DF.get_mo_eri is DF.ao2mo


def test_mp2_energy_emulated(emu_lib):
    """An RMP2 correlation energy from ao2mo((co, cv, co, cv)) equals the one from the oracle's tensor within 1e-10 Eh."""
    mol, d, B, ref, nao, mf = _h2o(emu_lib)
    nocc = mol.nelectron // 2
    co, cv = mf.mo_coeff[:, :nocc], mf.mo_coeff[:, nocc:]
    e = _mp2_energy(d.ao2mo((co, cv, co, cv)), mf.mo_energy, nocc)
    e_ref = _mp2_energy(_np_ao2mo(ref, nao, [co, cv, co, cv], False, False)[0], mf.mo_energy, nocc)
    assert e < -0.1 and abs(e - e_ref) < 1e-10, (e, e_ref)


def test_get_eri_emulated(emu_lib):
    """get_eri = get_ao_eri = restore(8, B^T B): the s8 triangle of the AO-pair matrix, in one band and in bands of 7 rows."""
    mol, d, B, ref, nao, mf = _h2o(emu_lib)
    npair = nao * (nao + 1) // 2
    i, j = np.tril_indices(npair)
    want = (B.T @ B)[i, j]
    got = d.get_eri()
    assert got.shape == (npair * (npair + 1) // 2,)
    assert abs(got - want).max() < 1e-12 * abs(want).max(), abs(got - want).max()
    assert abs(got - (ref.T @ ref)[i, j]).max() < 1e-9
    assert d.get_ao_eri == d.get_eri and DF.get_ao_eri is DF.get_eri
    _set_tile(d, 7)
    try:
        assert np.array_equal(d.get_eri(), got)
    finally:
        _set_tile(d, -1)


def test_bands_bit_identical_emulated(emu_lib):
    """Output bands of a few rows (several bands, copies through the pipeline) give the one-band result bit for bit, for a
    symmetric output (mirrored diagonal blocks) and a rectangular one."""
    mol, d, B, ref, nao, mf = _h2o(emu_lib)
    nocc = mol.nelectron // 2
    mo = mf.mo_coeff
    co, cv = mo[:, :nocc], mo[:, nocc:]
    one = [d.ao2mo(mo), d.ao2mo((co, cv, co, cv)), d.ao2mo((mo, cv, co, co))]
    for rows in (1, 5, 67):
        _set_tile(d, rows)
        try:
            many = [d.ao2mo(mo), d.ao2mo((co, cv, co, cv)), d.ao2mo((mo, cv, co, co))]
        finally:
            _set_tile(d, -1)
        for a, b in zip(one, many):
            assert np.array_equal(a, b), rows


def test_host_rows_emulated(emu_lib):
    """Rows forced into (pinned) host memory are staged through the copy buffers: ao2mo gives the all-device result bit for bit
    (L is made row by row); get_eri adds the host rows' part to the device rows' part, a different summation order."""
    mol, d, B, ref, nao, mf = _h2o(emu_lib)
    nocc = mol.nelectron // 2
    mo = mf.mo_coeff
    co, cv = mo[:, :nocc], mo[:, nocc:]
    naux = d.get_naoaux()
    want = [d.ao2mo((co, cv, co, cv)), d.ao2mo(mo[:, :8], compact=False), d.get_eri()]
    for cap in (0, naux // 3):
        h = DF(mol, AUX, libpath=emu_lib).set_device_rows(cap).build()
        assert h.row_split() == (cap, naux - cap)
        got = [h.ao2mo((co, cv, co, cv)), h.ao2mo(mo[:, :8], compact=False), h.get_eri()]
        assert np.array_equal(got[0], want[0]) and np.array_equal(got[1], want[1]), cap
        assert abs(got[2] - want[2]).max() < 1e-14 * abs(want[2]).max(), cap


def test_pair_screened_emulated(emu_lib):
    """A pair-screened tensor: the dropped columns act as exact zeros, as loop() returns them."""
    atom = 'O 0 0 0; H 0 -0.757 0.587; H 0 0.757 0.587; O 5 0 0; H 5 -0.757 0.587; H 5 0.757 0.587'
    mol = gto.M(atom=atom, basis='cc-pvdz')
    d = DF(mol, 'weigend', libpath=emu_lib, pair_tol=1e-8).build()
    ncol, npair = d.pair_stats()
    assert ncol < npair
    B = d._cderi
    ref, nao = O.cholesky_eri(mol, make_auxmol(mol, 'weigend'))
    rng = np.random.RandomState(3)
    c1, c2 = np.linalg.qr(rng.standard_normal((nao, 12)))[0][:, :5], rng.standard_normal((nao, 4))
    got = d.ao2mo((c1, c2, c1, c1))
    want, n1, n2 = _np_ao2mo(B, nao, [c1, c2, c1, c1], False, True)
    assert (abs(got - want) <= 1e-12 * np.outer(n1, n2)).all()
    # the oracle's dense tensor differs from the screened one by the dropped columns (2-norm < 1e-8 each)
    assert abs(got - _np_ao2mo(ref, nao, [c1, c2, c1, c1], False, True)[0]).max() < 1e-6
    i, j = np.tril_indices(npair)
    ge = d.get_eri()
    assert abs(ge - (B.T @ B)[i, j]).max() < 1e-12 * abs(ge).max()


def test_cartesian_emulated(emu_lib):
    """mol.cart = True: the coefficients run over the Cartesian AOs; against the Cartesian oracle's tensor."""
    import cart_oracle as C
    mol = gto.M(atom=H2O, basis='cc-pvdz', cart=True)
    d = DF(mol, AUX, libpath=emu_lib).build()
    B = d._cderi
    ref = C.cholesky_eri(mol, make_auxmol(mol, AUX))[0]
    nao = d.nao
    assert nao == 25 and B.shape[1] == nao * (nao + 1) // 2
    rng = np.random.RandomState(5)
    c = rng.standard_normal((nao, 9))
    cs = [c[:, :4], c[:, 4:], c[:, :4], c[:, 4:]]
    _check(d.ao2mo(cs), B, ref, nao, cs, False, False)
    _check(d.ao2mo(c[:, :6]), B, ref, nao, [c[:, :6]] * 4, True, True)
    with pytest.raises(ValueError):
        d.ao2mo(np.zeros((24, 3)))


def test_range_coulomb_and_assigned_emulated(emu_lib):
    """A range_coulomb(omega) child transforms its own tensor; an assigned _cderi is transformed as given."""
    mol, d, B, ref, nao, mf = _h2o(emu_lib)
    mo = mf.mo_coeff[:, :7]
    sr = DF(mol, 'weigend', libpath=emu_lib).range_coulomb(0.3)
    Bsr = sr._cderi
    ref_sr, _ = O.cholesky_eri(mol, make_auxmol(mol, 'weigend'), omega=0.3)
    _check(sr.ao2mo(mo), Bsr, ref_sr, nao, [mo] * 4, True, True)
    a = DF(mol, libpath=emu_lib)
    a._cderi = ref
    _check(a.ao2mo(mo, compact=False), ref, ref, nao, [mo] * 4, False, False)


def test_refused_inputs_emulated(emu_lib):
    """Sharded tensors, complex coefficients and coefficients over the wrong AO count are refused with a message."""
    mol, d, B, ref, nao, mf = _h2o(emu_lib)
    mo = mf.mo_coeff
    with pytest.raises(NotImplementedError, match='sharded'):
        DF(mol, AUX, libpath=emu_lib, shard=(0, 2)).ao2mo(mo)
    with pytest.raises(NotImplementedError, match='sharded'):
        DF(mol, AUX, libpath=emu_lib, shard=(0, 2)).get_eri()
    with pytest.raises(NotImplementedError, match='complex'):
        d.ao2mo(mo + 0j)
    with pytest.raises(ValueError, match='nao'):
        d.ao2mo(mo[:-1])
    with pytest.raises(ValueError, match='nao'):
        d.ao2mo((mo, mo, mo[1:], mo))
    assert d.ao2mo((mo[:, :0], mo, mo, mo)).shape == (0, nao * (nao + 1) // 2)
    h = d._handle
    assert h.lib.b200jk_df_set_ao2mo_tile(h._h, 0) != 0


# ---- GPU -------------------------------------------------------------------------------------------------------------------

@pytest.mark.gpu
def test_small_cases_gpu():
    """The emulated cases on sm_90a: orbital shapes, MP2 energy, get_eri, bands, host rows."""
    mol, d, B, ref, nao, mf = _h2o(None)
    nocc = mol.nelectron // 2
    mo = mf.mo_coeff
    _run_orbital_cases(d, B, ref, nao, mo, nocc)
    co, cv = mo[:, :nocc], mo[:, nocc:]
    ovov = d.ao2mo((co, cv, co, cv))
    e = _mp2_energy(ovov, mf.mo_energy, nocc)
    e_ref = _mp2_energy(_np_ao2mo(ref, nao, [co, cv, co, cv], False, False)[0], mf.mo_energy, nocc)
    assert abs(e - e_ref) < 1e-10, (e, e_ref)
    npair = nao * (nao + 1) // 2
    i, j = np.tril_indices(npair)
    ge = d.get_eri()
    assert abs(ge - (B.T @ B)[i, j]).max() < 1e-12 * abs(ge).max()
    full = d.ao2mo(mo)
    _set_tile(d, 5)
    try:
        assert abs(d.ao2mo(mo) - full).max() <= 1e-14 * abs(full).max()
        assert abs(d.get_eri() - ge).max() <= 1e-14 * abs(ge).max()
    finally:
        _set_tile(d, -1)
    h = DF(mol, AUX).set_device_rows(d.get_naoaux() // 3).build()
    try:
        assert np.array_equal(h.ao2mo((co, cv, co, cv)), ovov)
        assert abs(h.get_eri() - ge).max() < 1e-14 * abs(ge).max()
    finally:
        h.reset()
    t = d.ao2mo_times()
    assert t['total'] > 0 and t['stage2'] > 0, t


def _blocked_np(d, cs, s12, s34):
    """numpy transform of a large tensor read back row block by row block."""
    nao = d.nao
    L1, L2 = [], []
    for blk in d.loop(blksize=256):
        Bf = _unpack(blk, nao)
        L1.append(_half(Bf, cs[0], cs[1], s12))
        L2.append(_half(Bf, cs[2], cs[3], s34))
        del Bf
    L1, L2 = np.vstack(L1), np.vstack(L2)
    return L1.T @ L2, np.linalg.norm(L1, axis=0), np.linalg.norm(L2, axis=0)


def _check_blocked(d, got, cs, s12, s34):
    want, n1, n2 = _blocked_np(d, cs, s12, s34)
    err = abs(got - want) - 1e-12 * np.outer(n1, n2)
    assert got.shape == want.shape and (err <= 0).all(), err.max()


@pytest.mark.gpu
def test_benzene_tz_ovov_gpu():
    """benzene/cc-pVTZ: (ia|jb) over all occupied and virtual orbitals against numpy on the read-back tensor."""
    mol = gto.M(atom=geometry('benzene'), basis='cc-pvtz')
    d = DF(mol).build()
    try:
        nao = d.nao
        c = np.linalg.qr(np.random.RandomState(11).standard_normal((nao, nao)))[0]
        nocc = mol.nelectron // 2
        cs = [c[:, :nocc], c[:, nocc:], c[:, :nocc], c[:, nocc:]]
        got = d.ao2mo(cs)
        _check_blocked(d, got, cs, False, False)
        print('benzene/cc-pVTZ ovov %s: %s' % (got.shape, d.ao2mo_times()))
    finally:
        d.reset()


@pytest.mark.gpu
def test_c60_active_space_gpu():
    """C60/def2-SVP with 16 active orbitals: paaa ([mo, cas, cas, cas], compact=False, mcscf/df.py:140) and aaaa (mcscf/casci.py:373)
    against numpy on the read-back tensor."""
    mol = gto.M(atom=geometry('c60'), basis='def2-svp')
    d = DF(mol).build()
    try:
        nao = d.nao
        mo = np.linalg.qr(np.random.RandomState(13).standard_normal((nao, nao)))[0]
        nocc = mol.nelectron // 2
        cas = mo[:, nocc - 8:nocc + 8]
        paaa = d.ao2mo([mo, cas, cas, cas], compact=False)
        t1 = d.ao2mo_times()
        aaaa = d.ao2mo(cas)
        assert paaa.shape == (nao * 16, 256) and aaaa.shape == (136, 136)
        _check_blocked(d, paaa, [mo, cas, cas, cas], False, False)
        _check_blocked(d, aaaa, [cas] * 4, True, True)
        print('C60/def2-SVP paaa %s: %s; aaaa: %s' % (paaa.shape, t1, d.ao2mo_times()))
    finally:
        d.reset()
