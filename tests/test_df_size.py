"""Oracle parity of the density-fitting path AT THE SIZES of BASELINE.json configs 3-5 (C60/def2-SVP, Taxol/def2-TZVP, and
Taxol/def2-SVP, the largest of them that one 80 GB GPU holds;
(Gly)30 needs more than one GPU and is checked by bench.py's parity leg at N >= 4 with the same fixtures).

Fixtures: tests/golden/df_size_<name>.npz from tools/make_golden_df_size.py (CPU oracle): sampled AO-pair columns of the
tensor over ALL auxiliary rows, and J rows / K of a density supported on a few shells (exact from the oracle's shell slab).
Bar: 1e-9 Eh on J/K elements (north_star); tensor columns 1e-9 as well."""
import numpy as np
import pytest

import df_size_check as S
from pyscf_b200 import gto
from pyscf_b200.df import DF, TaggedDM
from pyscf_b200.gto.mole import geometry, make_auxmol

# taxol_svp: the Taxol tensor in def2-SVP (28 GB) fits one 80 GB GPU, the int8 slices of all its rows (51 GB) do not, so both
# the resident slices and the slices re-cut per call take part in every K build
CASES = {'c60': ('c60', 'def2-svp'), 'taxol': ('taxol', 'def2-tzvp'), 'taxol_svp': ('taxol', 'def2-svp'), 'gly4': ('gly4', 'cc-pvdz')}


def test_fixture_against_full_oracle_gly4():
    """The slab construction of the fixtures reproduces the oracle's full-tensor J/K (small molecule, CPU only)."""
    from oracle import oracle as O
    z = S.load('gly4')
    mol = gto.M(atom=geometry('gly4'), basis='cc-pvdz')
    cderi, nao = O.cholesky_eri(mol, make_auxmol(mol))
    assert abs(cderi[:, z['cols']] - z['cderi_cols']).max() < 1e-12
    c = S.slab_coeff(z)
    vj, vk = O.df_get_jk(cderi, nao, 2.0 * c.dot(c.T))
    r = S.compare_jk(z, vj, vk)
    assert r['max_abs_dJ'] < 1e-11 and r['max_abs_dK'] < 1e-11 and r['d_fp_K'] < 1e-10, r


@pytest.mark.gpu
@pytest.mark.parametrize('name', ['gly4', 'c60', 'taxol_svp', 'taxol'])
def test_df_parity_at_size(name):
    import torch
    z = S.load(name)
    assert z is not None, 'fixture missing: python tools/make_golden_df_size.py ' + name
    if name == 'taxol' and torch.cuda.get_device_properties(0).total_memory < 150e9:
        pytest.skip('the 111 GB Taxol tensor does not fit one GPU of %.0f GB' % (torch.cuda.get_device_properties(0).total_memory / 1e9))
    geom, basis = CASES[name]
    mol = gto.M(atom=geometry(geom), basis=basis)
    d = DF(mol).build()
    try:
        assert d.get_naoaux() == int(z['naux']) and mol.nao == int(z['nao'])
        dc = S.check_columns(d, z)
        assert dc < 1e-9, ('cderi columns', dc)
        c = S.slab_coeff(z)
        occ = np.full(c.shape[1], 2.0)
        dm = 2.0 * c.dot(c.T)
        # tensor-core engine (orbital tag, int8 slices) and the general-density engine on the bare matrix
        vj1, vk1 = d.get_jk(TaggedDM(dm, mo_coeff=c, mo_occ=occ), hermi=1)
        r1 = S.compare_jk(z, vj1, vk1)
        assert max(r1['max_abs_dJ'], r1['max_abs_dK'], r1['max_abs_dK_diag']) < 1e-9, ('orbital-tagged', r1)
        vj2, vk2 = d.get_jk(dm, hermi=1)
        r2 = S.compare_jk(z, vj2, vk2)
        assert max(r2['max_abs_dJ'], r2['max_abs_dK'], r2['max_abs_dK_diag']) < 1e-9, ('general density', r2)
        # SCF-like density of the bench: the two engines against each other on the same tensor
        rng = np.random.RandomState(1)
        co, _ = np.linalg.qr(rng.standard_normal((mol.nao, int(z['nocc']))))
        dms = 2.0 * co.dot(co.T)
        _, vk3 = d.get_jk(TaggedDM(dms, mo_coeff=co, mo_occ=np.full(co.shape[1], 2.0)), hermi=1, with_j=False)
        _, vk4 = d.get_jk(dms, hermi=1, with_j=False)
        assert abs(vk3 - vk4).max() < 1e-9, abs(vk3 - vk4).max()
        print('%s: cderi cols %.1e | tagged %s | general %s | engines %.1e' % (name, dc, r1, r2, abs(vk3 - vk4).max()))
    finally:
        d.reset()
