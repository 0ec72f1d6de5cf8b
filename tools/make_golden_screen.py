"""Stores what the reference's own C driver (oracle/_ref: CVHFnr_dm_cond, CVHFnrs8_prescreen and the J/K digestion, compiled
from the reference sources by oracle/Makefile.ref) computes with the screening at work, for the `chain` system and the two
densities of tests/screen_ref.py::golden_cases at direct_scf_tol 1e-13, 1e-9 and 1e-6:  tests/golden/screen_ref.npz.
test_model_against_oracle_and_reference_driver compares the screening model of tests/screen_ref.py with it."""
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, 'tests')]
from pyscf_b200 import gto  # noqa: E402
from oracle import ref_driver as R  # noqa: E402
import screen_ref as S  # noqa: E402

if not R.available():
    sys.exit('oracle/_ref is not built')
mol = gto.M(unit='Bohr', **S.CHAIN)
B = S.Basis(mol._atm, mol._bas, mol._env)
out = {}
for name, (dm, hermi) in S.golden_cases(B).items():
    out['%s_dm' % name], out['%s_hermi' % name] = dm, hermi
    for tol in S.TOLS:
        vj, vk = R.get_jk(mol, dm, hermi=hermi, direct_scf_tol=tol)
        out['%s_%g_vj' % (name, tol)], out['%s_%g_vk' % (name, tol)] = vj, vk
np.savez_compressed(os.path.join(ROOT, 'tests', 'golden', 'screen_ref.npz'), **out)
