"""Stores what the reference's own C driver (oracle/_ref, compiled from the reference sources by oracle/Makefile.ref)
computes for the inputs of tests/test_oracle_ref.py and the q_cond check of tests/test_host_emulation.py, so that those
tests compare against the reference without the reference tree:  tests/golden/ref_driver.npz."""
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from pyscf_b200 import gto  # noqa: E402
from oracle import ref_driver as R  # noqa: E402

H2O = 'O 0 0 0; H 0 -0.757 0.587; H 0 0.757 0.587'
if not R.available():
    sys.exit('oracle/_ref is not built')
out = {}
mol = gto.M(atom=H2O, basis='cc-pvdz')
nao = mol.nao
np.random.seed(1)
dm = np.random.random((nao, nao))
out['dz_vj'], out['dz_vk'] = R.get_jk(mol, dm, hermi=0)
out['dz_eye_vj'], out['dz_eye_vk'] = R.get_jk(mol, np.eye(nao), hermi=1)
mol = gto.M(atom=H2O, basis='cc-pvtz')
np.random.seed(4)
dm = np.random.random((2, mol.nao, mol.nao))
dm = dm + dm.transpose(0, 2, 1)
out['tz_vj'], out['tz_vk'] = R.get_jk(mol, dm, hermi=1)
out['tz_vj_sr'], out['tz_vk_sr'] = R.get_jk(mol, dm, hermi=1, omega=0.4)
mol = gto.M(atom='O 0 0 0; H 0 -0.757 0.587; H 0.3 0.757 0.587', basis='cc-pvtz')
out['q_cond_tz'] = R.q_cond(mol)
np.savez_compressed(os.path.join(ROOT, 'tests', 'golden', 'ref_driver.npz'), **out)
