"""The reference's own C driver/digestion agrees with the oracle's restatement and reproduces the reference fingerprints.
Its results are stored in tests/golden/ref_driver.npz (tools/make_golden_ref.py, from oracle/_ref compiled from the
reference sources); when oracle/_ref is built, the live driver is checked against the stored results as well."""
import os

import numpy as np

from pyscf_b200 import gto
from oracle import oracle as O
from oracle import ref_driver as R

H2O = 'O 0 0 0; H 0 -0.757 0.587; H 0 0.757 0.587'
GOLDEN = np.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), 'golden', 'ref_driver.npz'))


def _same_as_golden(key, v):
    if R.available():
        assert abs(v - GOLDEN[key]).max() < 1e-12, key


def test_reference_driver_fingerprints():
    mol = gto.M(atom=H2O, basis='cc-pvdz')
    nao = mol.nao
    vj, vk = GOLDEN['dz_vj'], GOLDEN['dz_vk']
    assert abs(np.linalg.norm(vj) - 77.035779188661465) < 1e-9      # pyscf/scf/test/test_rhf.py:908
    assert abs(O.fp(vk) - (-12.365527167710301)) < 1e-9             # :934
    vj, vk = GOLDEN['dz_eye_vj'], GOLDEN['dz_eye_vk']
    assert abs(O.fp(vj) - 1.6593323222866125) < 1e-9 and abs(O.fp(vk) - (-1.4662135224053987)) < 1e-9
    if R.available():
        np.random.seed(1)
        dm = np.random.random((nao, nao))
        for key, v in zip(('dz_vj', 'dz_vk'), R.get_jk(mol, dm, hermi=0)):
            _same_as_golden(key, v)
        for key, v in zip(('dz_eye_vj', 'dz_eye_vk'), R.get_jk(mol, np.eye(nao), hermi=1)):
            _same_as_golden(key, v)


def test_reference_driver_equals_oracle_driver():
    mol = gto.M(atom=H2O, basis='cc-pvtz')
    np.random.seed(4)
    dm = np.random.random((2, mol.nao, mol.nao))
    dm = dm + dm.transpose(0, 2, 1)
    vj, vk = GOLDEN['tz_vj'], GOLDEN['tz_vk']
    rj, rk = O.get_jk(mol, dm)
    assert abs(vj - rj).max() < 1e-11 and abs(vk - rk).max() < 1e-11
    vj, vk = GOLDEN['tz_vj_sr'], GOLDEN['tz_vk_sr']
    rj, rk = O.get_jk(mol, dm, omega=0.4)
    assert abs(vj - rj).max() < 1e-11 and abs(vk - rk).max() < 1e-11
    if R.available():
        for key, v in zip(('tz_vj', 'tz_vk'), R.get_jk(mol, dm, hermi=1)):
            _same_as_golden(key, v)
        for key, v in zip(('tz_vj_sr', 'tz_vk_sr'), R.get_jk(mol, dm, hermi=1, omega=0.4)):
            _same_as_golden(key, v)
