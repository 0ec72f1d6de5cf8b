"""Density-fitting path: emulated (CPU) and GPU parity against the oracle's restatement of
incore.cholesky_eri / df_jk.get_jk and the reference fingerprints (pyscf/df/test/test_df_jk.py:144-156)."""
import numpy as np
import pytest

from pyscf_b200 import gto
from pyscf_b200.df import DF, TaggedDM
from pyscf_b200.gto.mole import make_auxmol, geometry
from oracle import oracle as O

H2O = 'O 0 0 0; H 0 -0.757 0.587; H 0 0.757 0.587'


def _check_h2o(libpath):
    mol = gto.M(atom=H2O, basis='cc-pvdz')
    d = DF(mol, 'weigend', libpath=libpath).build()
    ref, nao = O.cholesky_eri(mol, make_auxmol(mol, 'weigend'))
    assert d.get_naoaux() == ref.shape[0]
    assert abs(d._cderi - ref).max() < 1e-10
    np.random.seed(1)
    dms = np.random.random((2, nao, nao))
    vj, vk = d.get_jk(dms, hermi=0)
    assert abs(O.fp(vj) - (-194.15910890730066)) < 1e-9   # test_df_jk.py:151-152
    assert abs(O.fp(vk) - (-46.365071587653517)) < 1e-9
    rj, rk = O.df_get_jk(ref, nao, dms)
    assert abs(vj - rj).max() < 1e-10 and abs(vk - rk).max() < 1e-10
    # mo_coeff fast path == general path (df_jk.py:339-357 vs :382-408)
    c = np.linalg.qr(np.random.random((nao, 5)))[0]
    occ = np.full(5, 2.0)
    dm = TaggedDM((c * occ).dot(c.T), mo_coeff=c, mo_occ=occ)
    vj1, vk1 = d.get_jk(dm, hermi=1)
    vj2, vk2 = d.get_jk(np.asarray(dm), hermi=1)
    assert abs(vj1 - vj2).max() < 1e-10 and abs(vk1 - vk2).max() < 1e-10
    return d


def test_df_emulated(emu_lib):
    _check_h2o(emu_lib)


def test_df_emulated_long_range(emu_lib):
    mol = gto.M(atom=H2O, basis='6-31g')
    d = DF(mol, 'weigend', libpath=emu_lib)
    d.omega = 0.3
    d.build()
    ref, nao = O.cholesky_eri(mol, make_auxmol(mol, 'weigend'), omega=0.3)
    # the long-range metric is numerically singular (smallest eigenvalue ~1e-15), so cderi itself is not
    # unique to rounding (SURVEY.md §7 hard part 6; the reference pins RSH-DF to 1e-3, df/test/test_df.py:101-117):
    # compare the J/K it produces
    np.random.seed(0)
    dm = np.random.random((nao, nao))
    dm = dm + dm.T
    vj, vk = d.get_jk(dm)
    rj, rk = O.df_get_jk(ref, nao, dm)
    assert abs(vj - rj).max() < 1e-8 and abs(vk - rk).max() < 1e-8


def test_df_long_range_k_against_exact_4center(emu_lib):
    """The reference pins RSH-DF only to 3 decimals (pyscf/df/test/test_df.py:101-117; SURVEY.md §8c): pin the long-range
    fitted J/K against the exact 4-center long-range J/K instead.  The erf-attenuated operator is smooth, so the auxiliary
    basis resolves it far better (5e-7 here) than the full Coulomb operator (3e-2 / 1e-1 with this J-fit basis)."""
    from pyscf_b200.jk import VHFOpt
    mol = gto.M(atom=H2O, basis='cc-pvdz')
    np.random.seed(0)
    dm = np.random.random((mol.nao, mol.nao))
    dm = dm + dm.T
    d = DF(mol, 'weigend', libpath=emu_lib).build()
    vj, vk = d.get_jk(dm, omega=0.3)                      # builds the omega tensor on demand (range_coulomb)
    ej, ek = VHFOpt(mol, omega=0.3, libpath=emu_lib).get_jk(dm)
    assert abs(vj - ej).max() < 1e-5 and abs(vk - ek).max() < 1e-5
    vj, vk = d.get_jk(dm)
    ej, ek = VHFOpt(mol, libpath=emu_lib).get_jk(dm)
    assert 1e-4 < abs(vk - ek).max() < 0.2 and abs(vj - ej).max() < 0.1   # fitting error of the full operator, for scale


def _check_orbital_sets(libpath):
    """Densities tagged with several orbital sets (UHF: one per spin; ROHF: one set, occupations 0/1/2 for an (alpha, beta)
    density pair), pyscf/df/df_jk.py:339-357: J for all densities at once, K per set through the occupied-orbital engine;
    must equal the general-density algebra."""
    mol = gto.M(atom=H2O, basis='cc-pvdz')
    nao = mol.nao
    d = DF(mol, 'weigend', libpath=libpath).build()
    ref, _ = O.cholesky_eri(mol, make_auxmol(mol, 'weigend'))
    rng = np.random.RandomState(7)
    ca = np.linalg.qr(rng.random_sample((nao, nao)))[0]
    cb = np.linalg.qr(rng.random_sample((nao, nao)))[0]
    occ_a = np.zeros(nao); occ_a[:5] = 1.0
    occ_b = np.zeros(nao); occ_b[:4] = 1.0                    # different numbers of occupied orbitals per spin
    dma = (ca * occ_a).dot(ca.T)
    dmb = (cb * occ_b).dot(cb.T)
    dms = np.array([dma, dmb])
    vj, vk = d.get_jk(TaggedDM(dms, mo_coeff=np.array([ca, cb]), mo_occ=np.array([occ_a, occ_b])))
    rj, rk = O.df_get_jk(ref, nao, dms)
    assert vj.shape == dms.shape and abs(vj - rj).max() < 1e-9 and abs(vk - rk).max() < 1e-9
    gj, gk = d.get_jk(dms)                                     # untagged: general-density path
    assert abs(vj - gj).max() < 1e-10 and abs(vk - gk).max() < 1e-10
    # ROHF: one orbital set with occupations 2,2,2,1,1,0,... for the (alpha, beta) densities
    occ = np.zeros(nao); occ[:3] = 2.0; occ[3:5] = 1.0
    da = (ca * (occ > 0)).dot(ca.T)
    db = (ca * (occ == 2)).dot(ca.T)
    pair = np.array([da, db])
    vj, vk = d.get_jk(TaggedDM(pair, mo_coeff=ca, mo_occ=occ))
    rj, rk = O.df_get_jk(ref, nao, pair)
    assert abs(vj - rj).max() < 1e-9 and abs(vk - rk).max() < 1e-9
    # fractional occupations scale the orbitals by sqrt(occ); a negative occupation falls back to the general path
    occ_f = np.zeros(nao); occ_f[:4] = [2.0, 1.5, 0.5, 0.25]
    df_ = (ca * occ_f).dot(ca.T)
    assert abs(d.get_jk(TaggedDM(df_, mo_coeff=ca, mo_occ=occ_f))[1] - O.df_get_jk(ref, nao, df_)[1]).max() < 1e-9
    occ_n = occ_f.copy(); occ_n[5] = -0.5
    dn = (ca * occ_n).dot(ca.T)
    assert abs(d.get_jk(TaggedDM(dn, mo_coeff=ca, mo_occ=occ_n))[1] - O.df_get_jk(ref, nao, dn)[1]).max() < 1e-9
    # K only, and an empty orbital set
    vj, vk = d.get_jk(TaggedDM(dms, mo_coeff=np.array([ca, cb]), mo_occ=np.array([occ_a, 0 * occ_b])), with_j=False)
    assert vj is None and abs(vk[0] - rk0(ref, nao, dma)).max() < 1e-9 and abs(vk[1]).max() == 0


def rk0(ref, nao, dm):
    return O.df_get_jk(ref, nao, dm)[1]


def test_orbital_sets_emulated(emu_lib):
    _check_orbital_sets(emu_lib)


@pytest.mark.gpu
def test_orbital_sets_gpu():
    _check_orbital_sets(None)


def _check_assign_cderi(libpath, tmpdir):
    """mf.with_df._cderi = ndarray (pyscf/df/df.py:116-118; pyscf/df/test/test_df_jk.py:135-142 assigns an exact factorisation
    of the 4-center integrals and recovers the non-DF energy): a tensor made elsewhere is uploaded instead of built."""
    import scipy.linalg
    mol = gto.M(atom=H2O, basis='6-31g')
    nao = mol.nao
    # (1) exact factorisation of (ij|kl): DF algebra on it must reproduce the exact 4-center J/K
    eri = O.int2e(mol)
    i, j = np.tril_indices(nao)
    e4 = eri[i, j][:, i, j]                      # aosym s4 as a (npair, npair) matrix
    w, u = scipy.linalg.eigh(e4)
    idx = w > 1e-9
    exact = (u[:, idx] * np.sqrt(w[idx])).T.copy()
    d = DF(mol, libpath=libpath)
    d._cderi = exact
    np.random.seed(5)
    dm = np.random.random((nao, nao))
    dm = dm + dm.T
    vj, vk = d.get_jk(dm)
    rj, rk = O.get_jk(mol, dm)
    assert d.get_naoaux() == exact.shape[0]
    assert abs(vj - rj).max() < 1e-7 and abs(vk - rk).max() < 1e-7          # eigenvalues below 1e-9 were dropped
    assert abs(d.get_j(dm) - vj).max() < 1e-12                                # J-only goes through the tensor
    c = np.linalg.qr(np.random.random((nao, 5)))[0]
    dmo = TaggedDM(2 * c.dot(c.T), mo_coeff=c, mo_occ=np.full(5, 2.0))
    assert abs(d.get_jk(dmo)[1] - O.get_jk(mol, np.asarray(dmo))[1]).max() < 1e-7   # orbital (tensor-core) K path
    # (2) round trip of a built tensor through a file: same J/K as the DF object that built it
    a = DF(mol, 'weigend', libpath=libpath).build()
    path = a.save(str(tmpdir / 'cderi.npy'))
    b = DF(mol, libpath=libpath)
    b._cderi = path
    ja, ka = a.get_jk(dm)
    jb, kb = b.get_jk(dm)
    assert abs(ja - jb).max() < 1e-12 and abs(ka - kb).max() < 1e-12
    assert abs(b._cderi - a._cderi).max() == 0
    # (3) row-sharded upload: every rank takes its rows of the assigned tensor, partial J/K add up
    parts = []
    for r in range(2):
        p = DF(mol, libpath=libpath, shard=(r, 2))
        p._cderi = path
        p.build()
        h = p._handle
        h.check(h.lib.b200jk_set_shard(h._h, r, 2), 'b200jk_set_shard')
        parts.append(p.get_jk(dm))
        assert sum(len(blk) for blk in p.loop()) in (a.get_naoaux() // 2, a.get_naoaux() - a.get_naoaux() // 2)
    assert abs(parts[0][0] + parts[1][0] - ja).max() < 1e-11 and abs(parts[0][1] + parts[1][1] - ka).max() < 1e-11
    with pytest.raises(RuntimeError):
        bad = DF(mol, libpath=libpath)
        bad._cderi = np.zeros((3, 7))
        bad.build()


def test_assign_cderi_emulated(emu_lib, tmp_path):
    _check_assign_cderi(emu_lib, tmp_path)


@pytest.mark.gpu
def test_assign_cderi_gpu(tmp_path):
    _check_assign_cderi(None, tmp_path)


def _check_direct_j(libpath):
    # integral-direct J (no tensor; df_jk.get_j, pyscf/df/df_jk.py:415-506) == J from the stored tensor;
    # reference fingerprint of the DF J matrix, pyscf/df/test/test_df_jk.py:151
    mol = gto.M(atom=H2O, basis='cc-pvdz')
    d = DF(mol, 'weigend', libpath=libpath)
    nao = mol.nao
    np.random.seed(1)
    dms = np.random.random((2, nao, nao))
    vj, vk = d.get_jk(dms, hermi=0, with_k=False)
    assert vk is None and d._handle is None          # no tensor was built
    assert abs(O.fp(vj) - (-194.15910890730066)) < 1e-9
    ref, _ = O.cholesky_eri(mol, make_auxmol(mol, 'weigend'))
    rj, _ = O.df_get_jk(ref, nao, dms)
    assert abs(vj - rj).max() < 1e-10
    # f orbital shells / g auxiliary shells, one non-symmetric density
    mol = gto.M(atom='He 0 0 0; Ne 1.2 0.3 0', basis='cc-pvtz')
    d = DF(mol, 'def2-universal-jkfit', libpath=libpath)
    dm = np.random.random((mol.nao, mol.nao))
    vj = d.get_j(dm)
    vj2 = d.build().get_jk(dm, hermi=0, with_k=False)[0]
    assert abs(vj - vj2).max() < 1e-9
    # RIJONX (only_dfj): J fitted, K exact (_DFHF.get_jk, pyscf/df/df_jk.py:157-179)
    from pyscf_b200.df import get_jk_only_dfj
    from pyscf_b200.jk import VHFOpt
    mol = gto.M(atom=H2O, basis='6-31g')
    d = DF(mol, 'weigend', libpath=libpath)
    dm = np.random.random((mol.nao, mol.nao))
    dm = dm + dm.T
    vj, vk = get_jk_only_dfj(d, mol, dm, vhfopt=VHFOpt(mol, libpath=libpath))
    ref, nao = O.cholesky_eri(mol, make_auxmol(mol, 'weigend'))
    assert abs(vj - O.df_get_jk(ref, nao, dm)[0]).max() < 1e-10
    assert abs(vk - O.get_jk(mol, dm)[1]).max() < 1e-10


def test_df_direct_j_emulated(emu_lib):
    _check_direct_j(emu_lib)


@pytest.mark.gpu
def test_df_direct_j_gpu():
    _check_direct_j(None)


@pytest.mark.gpu
def test_df_gpu_h2o():
    _check_h2o(None)


@pytest.mark.gpu
@pytest.mark.parametrize('basis,aux', [('cc-pvtz', 'cc-pvtz-jkfit'), ('def2-tzvp', 'def2-tzvp-jkfit')])
def test_df_gpu_high_l(basis, aux):
    # f orbital shells and g auxiliary shells
    mol = gto.M(atom=H2O, basis=basis)
    d = DF(mol, aux).build()
    ref, nao = O.cholesky_eri(mol, make_auxmol(mol, aux))
    assert abs(d._cderi - ref).max() < 1e-9
    np.random.seed(2)
    dm = np.random.random((nao, nao))
    dm = dm + dm.T
    vj, vk = d.get_jk(dm)
    rj, rk = O.df_get_jk(ref, nao, dm)
    assert abs(vj - rj).max() < 1e-9 and abs(vk - rk).max() < 1e-9


@pytest.mark.gpu
def test_df_gpu_benzene_properties():
    mol = gto.M(atom=geometry('benzene'), basis='def2-svp')
    d = DF(mol).build()          # def2-svp-jkfit via DEFAULT_AUXBASIS
    nao = mol.nao
    rng = np.random.RandomState(0)
    a = rng.random_sample((nao, nao)); a = a + a.T
    b = rng.random_sample((nao, nao)); b = b + b.T
    (ja, jb), (ka, kb) = d.get_jk(np.array([a, b]))
    jab, kab = d.get_jk(0.5 * a - 2 * b)
    assert abs(jab - (0.5 * ja - 2 * jb)).max() < 1e-9 and abs(kab - (0.5 * ka - 2 * kb)).max() < 1e-9
    assert abs(ja - ja.T).max() < 1e-10 and abs(ka - ka.T).max() < 1e-10
    # DF approximates the exact 4-center J/K from above in the Coulomb metric: compare loosely
    from pyscf_b200.jk import VHFOpt
    ej, ek = VHFOpt(mol).get_jk(a)
    assert abs(ja - ej).max() < 0.1 and abs(ka - ek).max() < 0.1   # fitting error of def2-svp-jkfit, elements O(100)
    # stage timers of the tensor-core K path (orbital-tagged density): every stage ran and was timed on the device
    c, _ = np.linalg.qr(rng.standard_normal((nao, 21)))
    from pyscf_b200.df import TaggedDM
    vj, vk = d.get_jk(TaggedDM(2 * c.dot(c.T), mo_coeff=c, mo_occ=np.full(21, 2.0)))
    st = d.stage_times()
    assert all(st[k][1] >= 1 and st[k][0] > 0 for k in ('j_rho', 'j_acc', 'k_gemm1', 'k_slice', 'k_gemm2')), st
    assert sum(v[0] for v in st.values()) <= d.stats()['ms_kernels'] * 1.05
    assert abs(vk - d.get_jk(2 * c.dot(c.T))[1]).max() < 1e-9      # int8 slices == FP64 general-density path


@pytest.mark.gpu
@pytest.mark.parametrize('name,geom,basis', [('gly4_dz', 'gly4', 'cc-pvdz'), ('bz_tz_df', 'benzene', 'cc-pvtz')])
def test_df_golden_vectors(name, geom, basis):
    """Oracle-generated fixtures (tools/make_golden_df.py): (Gly)4/cc-pVDZ is config 5's chemistry at oracle size (aux up
    to f), benzene/cc-pVTZ has f orbital and g auxiliary shells.  Tensor rows, fingerprint of the whole tensor, J and K
    (both K engines)."""
    import os
    g = np.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), 'golden', 'df_%s.npz' % name))
    mol = gto.M(atom=geometry(geom), basis=basis)
    d = DF(mol).build()
    assert d.get_naoaux() == int(g['naux'])
    cderi = d._cderi
    assert abs(cderi[g['rows']] - g['cderi_rows']).max() < 1e-9
    assert abs(O.fp(cderi) - float(g['fp_cderi'])) < 1e-8
    nao = mol.nao
    np.random.seed(1)
    dms = np.random.random((2, nao, nao))
    vj, vk = d.get_jk(dms, hermi=0)
    assert abs(vj - g['vj']).max() < 1e-9 and abs(vk - g['vk']).max() < 1e-9
    # occupied-orbital path through both K engines (int8 slices on the tensor cores, cuBLAS DGEMM)
    c = np.linalg.qr(np.random.random((nao, 21)))[0]
    occ = np.full(21, 2.0)
    dm = TaggedDM((c * occ).dot(c.T), mo_coeff=c, mo_occ=occ)
    k_tc = d.set_k_engine('tcgen05').get_jk(dm, with_j=False)[1]
    k_dg = d.set_k_engine('dgemm').get_jk(dm, with_j=False)[1]
    k_gen = d.get_jk(np.asarray(dm), hermi=1, with_j=False)[1]
    assert abs(k_tc - k_dg).max() < 1e-10 and abs(k_tc - k_gen).max() < 1e-10


@pytest.mark.gpu
@pytest.mark.parametrize('M,N,K,ns,sym', [(300, 77, 333, 7, 0), (65, 33, 129, 7, 0), (1, 200, 40, 7, 0), (257, 257, 130, 7, 1),
                                          (140, 95, 300, 3, 0), (129, 129, 256, 2, 1), (70, 45, 128, 8, 0), (33, 31, 17, 1, 0)])
def test_i8gemm_against_numpy(M, N, K, ns, sym):
    """The int8-slice tensor-core GEMM itself (b200jk_i8gemm_test: slicing + i8gemm_kernel, accumulate mode): C = A B^T with
    partial 128 x 32 tiles, K not a multiple of 128, 1..8 slices, and the upper-triangle-only symmetric mode (B = A)."""
    from pyscf_b200 import lib
    mol = gto.M(atom=H2O, basis='sto-3g')
    h = lib.Handle(mol._atm, mol._bas, np.array(mol._env, dtype=np.float64))
    rng = np.random.RandomState(M * 7 + N + ns)
    A = rng.standard_normal((M, K)) * np.exp(rng.uniform(-6, 6, (M, 1)))    # rows of very different magnitude
    B = A.copy() if sym else rng.standard_normal((N, K)) * np.exp(rng.uniform(-6, 6, (N, 1)))
    C = np.zeros((M, N))
    h.check(h.lib.b200jk_i8gemm_test(h._h, M, N, K, lib.dptr(A), lib.dptr(B), lib.dptr(C), ns, sym), 'b200jk_i8gemm_test')
    ref = A.dot(B.T)
    if sym:
        ref = np.triu(ref)
    # slicing error: every row to 2^-(6+7(ns-1)) of its largest element, pairs k + l >= ns dropped
    scale = abs(A).max(1)[:, None] * abs(B).max(1)[None, :] * K
    err = abs(C - ref) / scale
    assert err.max() < 2.0 ** (-(7 * ns - 3)), (err.max(), 2.0 ** (-(7 * ns - 3)))
    h.close()
