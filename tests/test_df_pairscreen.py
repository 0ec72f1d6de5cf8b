"""Pair-screened density-fitting tensors (DF(pair_tol=...), b200jk_df_set_pair_tol / b200jk_df_pair_stats): a row stores only the
AO-pair columns whose shell-pair Schwarz bound q = sqrt((ab|ab)) is >= pair_tol.

A dropped column has 2-norm <= q (||B[:, mu nu]||^2 = (mu nu|P) M^-1 (P|mu nu) <= (mu nu|mu nu)), which gives the bounds checked
here, with D~ the packed density (off-diagonal elements doubled) and rho = B D~ on the dense tensor:
  dropped output pair:  |J_mn| <= q_mn ||rho||_2                   (J of a dropped pair is 0)
  kept output pair:     |dJ_mn| <= q_mn sum_dropped q_ls |D~_ls|
  every pair:           |dK_mn| <= sum over (l, s) with (m l) or (s n) dropped of q_ml q_sn |D_ls|

CPU emulation: two H2O/cc-pVDZ 5 A apart and He-Ne/cc-pVTZ at 3.5 A, whose kept fractions lie between 30 and 90 %, and the
compact H2O/cc-pVDZ, where pair_tol = 1e-300 keeps every column and must reproduce the dense handle bit for bit.
GPU: C60/def2-SVP, Taxol/def2-TZVP and (Gly)30/cc-pVDZ (Coulomb and erf(0.3) tensors) on one GPU against the size fixtures."""
import numpy as np
import pytest

from pyscf_b200 import gto
from pyscf_b200.df import DF, TaggedDM
from pyscf_b200.gto.mole import geometry, make_auxmol
from pyscf_b200.jk import VHFOpt
from oracle import oracle as O

H2O = 'O 0 0 0; H 0 -0.757 0.587; H 0 0.757 0.587'
CASES = {'w2': ('O 0 0 0; H 0 -0.757 0.587; H 0 0.757 0.587; O 5 0 0; H 5 -0.757 0.587; H 5 0.757 0.587', 'cc-pvdz', 'weigend', 1e-8),
         'hene': ('He 0 0 0; Ne 3.5 0.3 0', 'cc-pvtz', 'def2-universal-jkfit', 1e-10)}


def _set_kblock(d, kb):
    h = d._handle
    h.check(h.lib.b200jk_df_set_kblock(h._h, int(kb), -1), 'b200jk_df_set_kblock')


def _inputs(nao, seed=1):
    """Two orbital-tagged densities, and two general densities with hermi 0 and 1 (n_dm = 2 in one call)."""
    rng = np.random.RandomState(seed)
    c1, c2 = (np.linalg.qr(rng.standard_normal((nao, 4)))[0] * np.sqrt(2.0) for _ in range(2))
    dm_g = rng.random_sample((2, nao, nao))
    dm_s = dm_g + dm_g.transpose(0, 2, 1)
    dms_t = np.array([c1 @ c1.T, c2 @ c2.T])
    return {'tagged': (TaggedDM(dms_t, mo_coeff=np.array([c1, c2]), mo_occ=np.full((2, 4), 1.0)), 1, dms_t),
            'general0': (dm_g, 0, dm_g), 'general1': (dm_s, 1, dm_s)}


def _segmented(mol):
    """The same basis with every general contraction split into its segments, one shell per contracted function, AO order
    unchanged: the shells whose bounds the selection uses (a reference shell's q_cond is the maximum over its segments)."""
    rows = []
    for b in mol._bas:
        for c in range(b[3]):
            r = b.copy()
            r[3] = 1
            r[6] = b[6] + c * b[2]
            rows.append(r)
    m = mol.copy()
    m._bas = np.array(rows, dtype=np.int32)
    m.nbas = len(rows)
    return m


def _ao_q(mol, q_shell):
    """Shell-pair bounds q_cond[nbas, nbas] expanded to AO pairs [nao, nao]."""
    loc = mol.ao_loc_nr()
    idx = np.repeat(np.arange(mol.nbas), np.diff(loc))
    return q_shell[np.ix_(idx, idx)]


def _tril(a):
    i, j = np.tril_indices(a.shape[-1])
    return a[..., i, j]


def _kept_mask(d, nao):
    """Kept packed columns of a screened handle, read through the interchange layout (a dropped column is exactly zero)."""
    full = d._cderi
    kept = (full != 0.0).any(axis=0)
    assert kept.sum() == d.pair_stats()[0]
    return full, kept


def _case(name, emu_lib, omega=None):
    atom, basis, aux, tol = CASES[name]
    mol = gto.M(atom=atom, basis=basis)
    auxmol = make_auxmol(mol, aux)
    ref, nao = O.cholesky_eri(mol, auxmol, omega=omega)
    seg = _segmented(mol)
    assert seg.nbas > mol.nbas          # the cases have general contractions
    q = _ao_q(seg, O.q_cond(seg, omega=omega))
    return mol, aux, tol, ref, nao, q


def _bounds(ref, q, kept_pk, dms):
    """Per-element bounds of |J - J_ref| and |K - K_ref| of a screened tensor (module docstring)."""
    nao = q.shape[0]
    kept = np.zeros((nao, nao), dtype=bool)
    i, j = np.tril_indices(nao)
    kept[i, j] = kept_pk
    kept[j, i] = kept_pk
    qd_pk = np.where(kept_pk, 0.0, _tril(q))
    bj, bk = [], []
    for dm in dms:
        dt = _tril(dm + dm.T) - 0.5 * _tril(np.diag(np.diag(dm + dm.T)))     # D~: diagonal once, off-diagonal doubled
        rho = ref @ dt
        jb = np.where(kept, q * (qd_pk @ abs(dt)), q * np.linalg.norm(rho))
        qk = np.where(kept, q, 0.0)
        ad = abs(dm)
        kb = q @ ad @ q - qk @ ad @ qk
        bj.append(jb)
        bk.append(np.maximum(kb, 0.0))
    return np.array(bj), np.array(bk)


def test_kept_set_is_the_schwarz_selection_emulated(emu_lib):
    """The kept columns are exactly the pairs with q_cond >= tol (the oracle's shell-pair bound, per segment of a general
    contraction), pairs within 1e-9 relative of tol aside, and the kept fraction is real sparsity (30 - 90 %)."""
    for name in CASES:
        mol, aux, tol, ref, nao, q = _case(name, emu_lib)
        d = DF(mol, aux, libpath=emu_lib, pair_tol=tol).build()
        ncol, npair = d.pair_stats()
        assert npair == nao * (nao + 1) // 2 and 0.3 < ncol / npair < 0.9, (name, ncol, npair)
        _, kept = _kept_mask(d, nao)
        qp = _tril(q)
        want = qp >= tol
        near = abs(qp / tol - 1.0) < 1e-9
        assert np.array_equal(kept[~near], want[~near]), name
        # a dropped column of the oracle's dense tensor is bounded by its q (and hence by tol)
        norms = np.linalg.norm(ref, axis=0)
        assert (norms[~kept] <= qp[~kept] * (1 + 1e-9) + 1e-15).all(), name
        assert (norms[~kept] < tol).all(), name


def test_identity_map_is_bit_identical_emulated(emu_lib, tmp_path):
    """pair_tol = 1e-300 on compact H2O keeps every column (ncol == npair, the map is the identity) and reproduces the dense handle
    bit for bit: J/K for tagged and general densities, hermi 0/1, n_dm = 2, both K engines' CPU algebra, loop(), cderi_columns(),
    save()."""
    mol = gto.M(atom=H2O, basis='cc-pvdz')
    nao = mol.nao
    d0 = DF(mol, 'weigend', libpath=emu_lib).build()
    d1 = DF(mol, 'weigend', libpath=emu_lib, pair_tol=1e-300).build()
    assert d1.pair_stats() == (nao * (nao + 1) // 2, nao * (nao + 1) // 2)
    assert d0.pair_stats() == d1.pair_stats()
    for kind, (dm, hermi, _) in _inputs(nao).items():
        a, b = d0.get_jk(dm, hermi=hermi), d1.get_jk(dm, hermi=hermi)
        assert np.array_equal(a[0], b[0]) and np.array_equal(a[1], b[1]), kind
    full = d0._cderi
    assert np.array_equal(np.vstack(list(d1.loop(blksize=7))), full)
    cols = np.array([0, 1, 5, 17, nao * (nao + 1) // 2 - 1])
    assert np.array_equal(d1.cderi_columns(cols), full[:, cols])
    assert np.array_equal(np.load(d1.save(str(tmp_path / 'c.npy'))), full)


@pytest.mark.parametrize('name', list(CASES))
def test_screened_tensor_and_jk_emulated(emu_lib, name):
    """Kept columns equal the dense tensor bit for bit and dropped ones are exactly 0; J/K deviate from the oracle's dense DF
    J/K by no more than the bounds of the module docstring."""
    mol, aux, tol, ref, nao, q = _case(name, emu_lib)
    dense = DF(mol, aux, libpath=emu_lib).build()._cderi
    d = DF(mol, aux, libpath=emu_lib, pair_tol=tol).build()
    full, kept = _kept_mask(d, nao)
    assert np.array_equal(full[:, kept], dense[:, kept]) and not full[:, ~kept].any()
    cols = np.flatnonzero(~kept)[:5].tolist() + np.flatnonzero(kept)[:5].tolist()
    assert np.array_equal(d.cderi_columns(cols), full[:, cols])
    for kind, (dm, hermi, dms) in _inputs(nao).items():
        vj, vk = d.get_jk(dm, hermi=hermi)
        rj, rk = O.df_get_jk(ref, nao, dms)
        bj, bk = _bounds(ref, q, kept, dms)
        assert (abs(vj - rj) <= bj + 1e-10).all(), (kind, (abs(vj - rj) - bj).max())
        assert (abs(vk - rk) <= bk + 1e-10).all(), (kind, (abs(vk - rk) - bk).max())
        assert abs(vj - rj).max() > 0 or kind == 'tagged'      # the screening is visible


@pytest.mark.parametrize('name', list(CASES))
def test_screened_split_emulated(emu_lib, name):
    """Forced device rows 0, 1 and naux/3 with a few rows per K block match the resident screened handle to 1e-12; host rows
    are stored and streamed at the screened row length."""
    mol, aux, tol, ref, nao, q = _case(name, emu_lib)
    d0 = DF(mol, aux, libpath=emu_lib, pair_tol=tol).build()
    naux = d0.get_naoaux()
    ncol = d0.pair_stats()[0]
    inputs = _inputs(nao)
    want = {k: d0.get_jk(v[0], hermi=v[1]) for k, v in inputs.items()}
    full = d0._cderi
    for cap in (0, 1, naux // 3):
        d = DF(mol, aux, libpath=emu_lib, pair_tol=tol).set_device_rows(cap).build()
        assert d.row_split() == (cap, naux - cap) and d.pair_stats()[0] == ncol
        _set_kblock(d, max(1, (naux - cap) // 7))
        for kind, (dm, hermi, _) in inputs.items():
            vj, vk = d.get_jk(dm, hermi=hermi)
            assert abs(vj - want[kind][0]).max() < 1e-12 and abs(vk - want[kind][1]).max() < 1e-12, (cap, kind)
        assert d.stream_stats()['bytes'] == (naux - cap) * ncol * 8
        assert np.array_equal(d._cderi, full)


def test_screened_sharded_emulated(emu_lib):
    """Two ranks arrive at the same columns, and their partial J/K sum to the unsharded screened result."""
    mol, aux, tol, ref, nao, q = _case('hene', emu_lib)
    d0 = DF(mol, aux, libpath=emu_lib, pair_tol=tol).build()
    dm = _inputs(nao)['general0'][0]
    wj, wk = d0.get_jk(dm, hermi=0)
    vj, vk = np.zeros_like(wj), np.zeros_like(wk)
    rows = []
    for rank in range(2):
        d = DF(mol, aux, libpath=emu_lib, shard=(rank, 2), pair_tol=tol).set_device_rows(3).build()
        assert d.pair_stats() == d0.pair_stats()
        _set_kblock(d, 4)
        pj, pk = d.get_jk(dm, hermi=0)
        vj += pj
        vk += pk
        rows.append(d._cderi)
    assert abs(vj - wj).max() < 1e-12 and abs(vk - wk).max() < 1e-12
    assert np.array_equal(np.vstack(rows), d0._cderi)


def test_range_coulomb_child_screened_with_its_operator_emulated(emu_lib):
    """A range_coulomb child inherits pair_tol and selects its columns with the erf-attenuated bound, which is never larger than
    the Coulomb one; its K stays within the bound against the oracle's erf tensor."""
    omega = 0.3
    mol, aux, tol, ref, nao, q = _case('w2', emu_lib, omega=omega)
    d = DF(mol, aux, libpath=emu_lib, pair_tol=tol).build()
    child = d.range_coulomb(omega)
    assert child.pair_tol == tol
    full, kept = _kept_mask(child, nao)
    qp = _tril(q)
    near = abs(qp / tol - 1.0) < 1e-9
    assert np.array_equal(kept[~near], (qp >= tol)[~near])
    assert child.pair_stats()[0] <= d.pair_stats()[0]
    assert not (kept & ~_kept_mask(d, nao)[1]).any()
    # the erf metric is poorly conditioned: the screening error is measured against the dense erf tensor of this library, whose
    # kept columns the screened one reproduces bit for bit
    dense = DF(mol, aux, libpath=emu_lib).range_coulomb(omega)
    assert np.array_equal(full[:, kept], dense._cderi[:, kept])
    for kind, (dm, hermi, dms) in _inputs(nao).items():
        _, vk = child.get_jk(dm, hermi=hermi, with_j=False)
        _, rk = dense.get_jk(dm, hermi=hermi, with_j=False)
        _, bk = _bounds(dense._cderi, q, kept, dms)
        assert (abs(vk - rk) <= bk + 1e-12).all(), kind
        assert abs(vk - rk).max() > 0


def test_setting_kept_by_reset_and_not_applied_to_assigned_tensor(emu_lib):
    """reset() keeps pair_tol; a tensor assigned through _cderi stays dense whatever pair_tol says."""
    mol, aux, tol, ref, nao, q = _case('hene', emu_lib)
    d = DF(mol, aux, libpath=emu_lib, pair_tol=tol).build()
    ncol = d.pair_stats()[0]
    d.reset()
    assert d.pair_tol == tol and d.pair_stats()[0] == ncol
    dense = DF(mol, aux, libpath=emu_lib).build()._cderi
    a = DF(mol, aux, libpath=emu_lib, pair_tol=tol)
    a._cderi = dense
    npair = nao * (nao + 1) // 2
    assert a.pair_stats() == (npair, npair)
    assert np.array_equal(a._cderi, dense)


# ---- GPU -------------------------------------------------------------------------------------------------------------------

def _check_fixture_columns(S, z, d, mol, q_shell):
    """Fixture columns: within 1e-9 where kept; exactly 0 where dropped, and the oracle column's 2-norm <= q there.  Shell pairs
    without a surviving primitive pair have q_cond 1e-100 and are not integrated by the dense build either: their oracle columns
    are below 1e-12.  A fixture made with the eigen-decomposed metric defines its rows only up to rotations (df_size_check), so
    only the rotation-invariant column norms of its dropped columns are checked."""
    got = d.cderi_columns(z['cols'])
    ref = z['cderi_cols']
    kept = (got != 0.0).any(axis=0)
    q = _tril(_ao_q(mol, q_shell))[z['cols']]
    unique = not ('chol' in z and int(z['chol']) == 0)
    dk = float(abs(got[:, kept] - ref[:, kept]).max()) if kept.any() and unique else None
    assert dk is None or dk < 1e-9, dk
    nd = np.linalg.norm(ref[:, ~kept], axis=0)
    assert (nd <= np.maximum(q[~kept] * (1 + 1e-9), 1e-12)).all(), (nd - q[~kept]).max()
    return dk, int((~kept).sum())


def _check_jk_fixture(S, z, d, mol, engines):
    c = S.slab_coeff(z)
    occ = np.full(c.shape[1], 2.0)
    dm = 2.0 * c.dot(c.T)
    out = {}
    for eng in engines:
        d.set_k_engine(eng, 7)
        vj1, vk1 = d.get_jk(TaggedDM(dm, mo_coeff=c, mo_occ=occ), hermi=1)
        r1 = S.compare_jk(z, vj1, vk1)
        assert max(r1['max_abs_dJ'], r1['max_abs_dK'], r1['max_abs_dK_diag']) < 1e-9, (eng, 'orbital-tagged', r1)
        vj2, vk2 = d.get_jk(dm, hermi=1)
        r2 = S.compare_jk(z, vj2, vk2)
        assert max(r2['max_abs_dJ'], r2['max_abs_dK'], r2['max_abs_dK_diag']) < 1e-9, (eng, 'general density', r2)
        out[eng] = (vj1, vk1, vj2, vk2)
    d.set_k_engine('tcgen05', 7)
    return out


@pytest.mark.gpu
def test_c60_identity_map_gpu():
    """C60/def2-SVP with pair_tol = 1e-300: every shell pair with a surviving primitive pair is kept.  The others (17 % of the
    columns of C60) are never columns; their dense columns are exactly zero, so the mapped kernels (column gather of DF-J, mapped
    rowexp / slicing / unpacking of DF-K) must give the dense build's results for both K engines.  The sampled tensor columns are
    bit-identical; J/K agree to 1e-12, the reordering freedom of the atomic accumulation of rho."""
    mol = gto.M(atom=geometry('c60'), basis='def2-svp')
    nao = mol.nao
    c = np.linalg.qr(np.random.RandomState(1).standard_normal((nao, 180)))[0]
    dm = 2.0 * c @ c.T
    inputs = [(TaggedDM(dm, mo_coeff=c, mo_occ=np.full(180, 2.0)), 1), (dm, 1), (np.random.RandomState(2).random_sample((nao, nao)), 0)]
    res, stats = [], []
    for tol in (None, 1e-300):
        d = DF(mol, pair_tol=tol).build()
        try:
            ncol, npair = d.pair_stats()
            stats.append((ncol, npair))
            out = [d.cderi_columns(np.arange(0, npair, 97))]
            for eng in ('tcgen05', 'dgemm'):
                d.set_k_engine(eng, 7)
                for dmi, hermi in inputs:
                    out.extend(d.get_jk(dmi, hermi=hermi))
            res.append(out)
        finally:
            d.reset()
    assert stats[0][0] == stats[0][1] and 0.5 < stats[1][0] / stats[1][1] < 1.0, stats
    dropped = ~(res[1][0] != 0.0).any(axis=0)
    assert dropped.any() and np.array_equal(res[0][0], res[1][0])      # dense columns of never-integrated pairs are exact zeros
    for i, (a, b) in enumerate(zip(res[0][1:], res[1][1:])):
        assert abs(a - b).max() < 1e-12, (i, abs(a - b).max())
    print('c60 pair_tol=1e-300: %d of %d columns, max |d| J/K %.1e'
          % (stats[1][0], stats[1][1], max(abs(a - b).max() for a, b in zip(res[0][1:], res[1][1:]))))


@pytest.mark.gpu
@pytest.mark.parametrize('split', ['resident', 'half_host'])
def test_c60_screened_gpu(split):
    """C60/def2-SVP at pair_tol = 1e-13 against the size fixture to 1e-9 with both K engines, all resident and with half of the
    rows in pinned host memory."""
    import df_size_check as S
    z = S.load('c60')
    mol = gto.M(atom=geometry('c60'), basis='def2-svp')
    q_shell = VHFOpt(mol).q_cond
    d = DF(mol, pair_tol=1e-13)
    if split == 'half_host':
        d.set_device_rows(int(z['naux']) // 2)
    d.build()
    try:
        ncol, npair = d.pair_stats()
        n_dev, n_host = d.row_split()
        if split == 'half_host':
            assert n_host > 0
        dk, ndrop = _check_fixture_columns(S, z, d, mol, q_shell)
        _check_jk_fixture(S, z, d, mol, ('tcgen05', 'dgemm'))
        print('c60 %s: kept %d of %d columns (%.1f %%), split %s, fixture cols %s (%d dropped), stream %s'
              % (split, ncol, npair, 100.0 * ncol / npair, (n_dev, n_host), dk, ndrop, d.stream_stats()))
    finally:
        d.reset()


@pytest.mark.gpu
def test_taxol_tzvp_screened_gpu():
    """Taxol/def2-TZVP at pair_tol = 1e-13 on one GPU against the size fixture to 1e-9."""
    import df_size_check as S
    z = S.load('taxol')
    mol = gto.M(atom=geometry('taxol'), basis='def2-tzvp')
    q_shell = VHFOpt(mol).q_cond
    d = DF(mol, pair_tol=1e-13).build()
    try:
        ncol, npair = d.pair_stats()
        dk, ndrop = _check_fixture_columns(S, z, d, mol, q_shell)
        _check_jk_fixture(S, z, d, mol, ('tcgen05',))
        print('taxol/def2-tzvp: kept %d of %d columns (%.1f %%, %.1f GB), split %s, fixture cols %s (%d dropped), stream %s'
              % (ncol, npair, 100.0 * ncol / npair, d.get_naoaux() * ncol * 8 / 1e9, d.row_split(), dk, ndrop, d.stream_stats()))
    finally:
        d.reset()


@pytest.mark.gpu
def test_gly30_wb97x_one_gpu():
    """(Gly)30/cc-pVDZ on ONE GPU at pair_tol = 1e-13: the Coulomb tensor and its range_coulomb(0.3) child, get_jk and
    get_k(omega=0.3) against df_size_gly30 / df_size_gly30_lr to 1e-9."""
    import df_size_check as S
    z, zlr = S.load('gly30'), S.load('gly30_lr')
    mol = gto.M(atom=geometry('gly30'), basis='cc-pvdz')
    d = DF(mol, pair_tol=1e-13).build()
    try:
        lr = d.range_coulomb(0.3)
        for name, t in (('coulomb', d), ('erf(0.3)', lr)):
            ncol, npair = t.pair_stats()
            print('gly30 %s: kept %d of %d columns (%.1f %%, %.1f GB), row split %s'
                  % (name, ncol, npair, 100.0 * ncol / npair, t.get_naoaux() * ncol * 8 / 1e9, t.row_split()))
        dk, ndrop = _check_fixture_columns(S, z, d, mol, VHFOpt(mol).q_cond)
        dk2, ndrop2 = _check_fixture_columns(S, zlr, lr, mol, VHFOpt(mol, omega=0.3).q_cond)
        c = S.slab_coeff(z)
        dm = 2.0 * c.dot(c.T)
        for tag, dmi in (('orbital-tagged', TaggedDM(dm, mo_coeff=c, mo_occ=np.full(c.shape[1], 2.0))), ('general density', dm)):
            vj, vk = d.get_jk(dmi, hermi=1)
            r = S.compare_jk(z, vj, vk)
            assert max(r['max_abs_dJ'], r['max_abs_dK'], r['max_abs_dK_diag']) < 1e-9, (tag, r)
            _, vklr = d.get_jk(dmi, hermi=1, with_j=False, omega=0.3)
            rl = S.compare_jk(zlr, None, vklr)
            assert max(rl['max_abs_dK'], rl['max_abs_dK_diag']) < 1e-9, (tag, 'long range', rl)
            print('gly30 %s: %s, long-range K %s' % (tag, r, rl))
        print('gly30 fixture columns: coulomb %s (%d dropped), erf %s (%d dropped)' % (dk, ndrop, dk2, ndrop2))
    finally:
        d.reset()
