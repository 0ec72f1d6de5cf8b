"""Converged SCF energies through the GPU J/K builders equal the reference's published values
(north_star: "converged SCF energy identical to reference tolerance").
  RHF  H2O/cc-pVDZ            -76.026765673119627   pyscf/scf/test/test_rhf.py:371-372
  DF-RHF H2O/cc-pVDZ/weigend  -76.025936299702536   pyscf/df/test/test_df_jk.py:57-59
One-electron matrices come from the CPU oracle (host-side, out of the GPU path's scope)."""
import numpy as np
import pytest

from pyscf_b200 import gto
from pyscf_b200.df import DF, TaggedDM
from pyscf_b200.jk import VHFOpt
from pyscf_b200.scf import RHF
from oracle import oracle as O

H2O = 'O 0 0 0; H 0 -0.757 0.587; H 0 0.757 0.587'


def _run(libpath, use_df):
    mol = gto.M(atom=H2O, basis='cc-pvdz')
    s = O.int1e(mol, 'ovlp')
    h = O.int1e(mol, 'kin') + O.int1e(mol, 'nuc')
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


def test_rhf_energy_emulated(emu_lib):
    e, ok = _run(emu_lib, False)
    assert ok and abs(e - (-76.026765673119627)) < 1e-8


def test_df_rhf_energy_emulated(emu_lib):
    e, ok = _run(emu_lib, True)
    assert ok and abs(e - (-76.025936299702536)) < 1e-8


@pytest.mark.gpu
def test_rhf_energy_gpu():
    e, ok = _run(None, False)
    assert ok and abs(e - (-76.026765673119627)) < 1e-8


@pytest.mark.gpu
def test_df_rhf_energy_gpu():
    e, ok = _run(None, True)
    assert ok and abs(e - (-76.025936299702536)) < 1e-8
