"""The sub-warp-per-quartet kernel family (pyscf_b200/csrc/jk_swq.cuh): which classes run on it, and its arithmetic on a case
where the lanes of one warp diverge in what they do.

A quartet of these classes is shared by T = 2, 4 or 8 consecutive lanes that walk the same kets, so a warp holds 4 to 16
quartets at once.  The J/K case below mixes, inside one warp, kept and screened-out quartets (two fragments 8 Angstrom apart,
a small density) and kets of different primitive counts (contracted carbon shells next to single-primitive hydrogen shells),
with three density matrices and hermi = 0 so that neither the J[ij] registers nor a symmetric K can hide a wrong segment."""
import ctypes

import numpy as np
import pytest

from pyscf_b200 import gto
from pyscf_b200.jk import VHFOpt
from oracle import oracle as O

from test_rys_eri import ALL_CLASSES, PAIR_ID, class_name, family, launched

# the sub-warp classes as launched (bra | ket) in pair-class ids: (dp|ps) (ds|pp) (dp|ds) (fs|ds) (fp|ps) (dd|ps) (pp|fs) (pp|pp)
SWQ = {(4, 1), (3, 2), (4, 3), (6, 3), (7, 1), (5, 1), (2, 6), (2, 2)}

GEOM = 'C 0 0 0; H 0 0.95 0.55; O 0 -0.7 0.9; C 0.3 0.2 8.0; H 0.3 1.2 8.1'


def launch_families(libpath):
    opt = VHFOpt(gto.M(atom='He 0 0 0', basis='sto-3g'), libpath=libpath)
    h = opt.handle
    fam = {}
    for cb in range(10):
        for ck in range(cb + 1):
            buf = (ctypes.c_int * 9)()
            assert h.lib.b200jk_class_launch_info(h._h, cb, ck, buf, 9) == 0
            fam[launched(cb, ck)] = buf[0]
    opt.close()
    return fam


def test_swq_classes(emu_lib):
    fam = launch_families(emu_lib)
    assert set(fam) == set(ALL_CLASSES)
    assert {c for c, f in fam.items() if f == 2} == SWQ, sorted(class_name(c) for c, f in fam.items() if f == 2)
    assert {c for c, f in fam.items() if f == 0} == {c for c in ALL_CLASSES if family(c) == 'tpq'}
    assert sum(f == 0 for f in fam.values()) == 12
    assert all(f == 1 for c, f in fam.items() if c not in SWQ and family(c) != 'tpq')
    # the slattice case of test_screening drives the block kernels' sub-chunk walk through (dd|ss)
    assert fam[launched(int(PAIR_ID(2, 2)), 0)] == 1


def mixed_case():
    mol = gto.M(atom=GEOM, basis='cc-pvtz')
    rng = np.random.RandomState(7)
    dms = rng.standard_normal((3, mol.nao, mol.nao)) * 1e-2
    dms[2] = dms[2] - dms[2].T        # an antisymmetric K density next to two general ones
    return mol, dms


def check_mixed(libpath):
    mol, dms = mixed_case()
    opt = VHFOpt(mol, libpath=libpath)
    vj, vk = opt.get_jk(dms, hermi=0)
    st = opt.stats()
    opt.close()
    rj, rk = O.get_jk(mol, dms, screen=False)
    assert abs(vj - rj).max() < 1e-10 and abs(vk - rk).max() < 1e-10, (abs(vj - rj).max(), abs(vk - rk).max())
    return st


def test_swq_mixed_warp_emulated(emu_lib):
    check_mixed(emu_lib)


@pytest.mark.gpu
def test_swq_mixed_warp_gpu():
    check_mixed(None)
