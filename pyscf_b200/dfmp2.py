"""DF-MP2 on the GPU from the resident density-fitting tensor: the DFRMP2 / DFUMP2 kernels (pyscf/mp/dfmp2.py:39-121,
pyscf/mp/dfump2.py:38-166) without forming (ia|jb) anywhere but pair by pair on the device.

  * kernel(with_df, occ_coeff, vir_coeff, occ_energy, vir_energy, with_t2)       RMP2: (e_corr, t2 [nocc, nocc, nvir, nvir])
  * ukernel(with_df, occ_coeffs, vir_coeffs, occ_energies, vir_energies, with_t2) UMP2: (e_corr, (t2aa, t2ab, t2bb))
  * patch(pt)   route a PySCF DFRMP2 / DFUMP2 instance whose with_df is a pyscf_b200.df.DF through the kernels above

e_corr is a float tagged with e_corr_ss and e_corr_os, the role of lib.tag_array in dfmp2.py:119.  The half-transformed
L[P, i nvir + a] of each spin is made on the device from the tensor rows (host-resident rows included) and the pair energies
are reduced there in a fixed order; only the energies and, with with_t2, the amplitudes come back (b200jk_df_mp2, df_mp2.cuh).
This module does not import pyscf: patch() only replaces two methods of the instance it is given.
"""
import numpy as np

from . import lib as _lib
from .df import _check_df, _coeff, _eris_ao2mo, _times

_T2_MEMORY_MSG = 'Insufficient memory for holding t2 incore. Please rerun with `with_t2 = False`.'   # dfmp2.py:59-61


class TaggedFloat(float):
    """A float carrying e_corr_ss and e_corr_os (lib.tag_array(emp2, e_corr_ss=..., e_corr_os=...), dfmp2.py:119)."""

    def __new__(cls, value, e_corr_ss, e_corr_os):
        x = float.__new__(cls, value)
        x.e_corr_ss = float(e_corr_ss)
        x.e_corr_os = float(e_corr_os)
        return x


def _energy(e, n, what):
    e = np.ascontiguousarray(np.asarray(e, dtype=np.float64).ravel())
    if len(e) != n:
        raise ValueError('DF-MP2: %d %s orbital energies for %d orbitals' % (len(e), what, n))
    return e


def _run(with_df, cos, cvs, eos, evs, t2_shapes):
    """b200jk_df_mp2 over nspin = len(cos) spins; t2_shapes: None or the shapes of the amplitude blocks to return."""
    nao = _check_df(with_df, 'DF-MP2', 'the pair energies are not linear in the local rows')
    ns = len(cos)
    cos = [_coeff(c, nao, 'occupied', 'DF-MP2') for c in cos]
    cvs = [_coeff(c, nao, 'virtual', 'DF-MP2') for c in cvs]
    nocc = np.array([c.shape[1] for c in cos], dtype=np.int32)
    nvir = np.array([c.shape[1] for c in cvs], dtype=np.int32)
    eos = [_energy(e, n, 'occupied') for e, n in zip(eos, nocc)]
    evs = [_energy(e, n, 'virtual') for e, n in zip(evs, nvir)]
    arr = _lib.c_double_p * ns
    t2 = None if t2_shapes is None else tuple(np.zeros(s) for s in t2_shapes)
    t2p = None if t2 is None else (_lib.c_double_p * len(t2))(*[_lib.dptr(x) for x in t2])
    e = np.zeros(2)
    h = with_df._handle
    h.check(h.lib.b200jk_df_mp2(h._h, ns, arr(*[_lib.dptr(c) for c in cos]), _lib.iptr(nocc), arr(*[_lib.dptr(c) for c in cvs]),
                                _lib.iptr(nvir), arr(*[_lib.dptr(x) for x in eos]), arr(*[_lib.dptr(x) for x in evs]),
                                _lib.dptr(e), t2p), 'b200jk_df_mp2')
    return TaggedFloat(e[0] + e[1], e[0], e[1]), t2


def kernel(with_df, occ_coeff, vir_coeff, occ_energy, vir_energy, with_t2=False):
    """RMP2 correlation energy (dfmp2.kernel): e_corr = e_corr_ss + e_corr_os with e_ss = ed + ex, e_os = ed (dfmp2.py:109-119);
    t2[i, j, a, b] = (ia|jb) / (e_i + e_j - e_a - e_b) when with_t2, else None."""
    no, nv = np.shape(occ_coeff)[-1], np.shape(vir_coeff)[-1]
    e, t2 = _run(with_df, [occ_coeff], [vir_coeff], [occ_energy], [vir_energy], [(no, no, nv, nv)] if with_t2 else None)
    return e, (None if t2 is None else t2[0])


def ukernel(with_df, occ_coeffs, vir_coeffs, occ_energies, vir_energies, with_t2=False):
    """UMP2 correlation energy (dfump2.kernel): e_ss = sum over spins of (ed + ex) / 2, e_os = ed of the alpha-beta pairs
    (dfump2.py:119,154,164); t2 = (aa, ab, bb) as dfump2.py:51-54 when with_t2, else None."""
    no = [np.shape(c)[-1] for c in occ_coeffs]
    nv = [np.shape(c)[-1] for c in vir_coeffs]
    shapes = [(no[0], no[0], nv[0], nv[0]), (no[0], no[1], nv[0], nv[1]), (no[1], no[1], nv[1], nv[1])]
    return _run(with_df, list(occ_coeffs), list(vir_coeffs), list(occ_energies), list(vir_energies), shapes if with_t2 else None)


def patch(pt):
    """Route a PySCF DFRMP2 / DFUMP2 instance whose with_df is a pyscf_b200.df.DF through the GPU kernels: pt.ao2mo and
    pt.init_amps are replaced on the instance, everything else (get_mo_energy, e_hf, frozen orbitals through split_mo_coeff /
    split_mo_energy, SCS, make_rdm1 on the returned t2, _finalize) stays PySCF's.  Returns pt."""
    def init_amps(mo_energy=None, mo_coeff=None, eris=None, with_t2=True):
        if eris is None:
            eris = pt.ao2mo(mo_coeff)
        if with_t2:
            no, nv = [int(x) for x in np.atleast_1d(eris.nocc)], [int(x) for x in np.atleast_1d(eris.nvir)]
            if eris.unrestricted:
                n = no[0] ** 2 * nv[0] ** 2 + no[0] * no[1] * nv[0] * nv[1] + no[1] ** 2 * nv[1] ** 2
            else:
                n = no[0] ** 2 * nv[0] ** 2
            if n * 8 / 1e6 > pt.max_memory:
                raise MemoryError(_T2_MEMORY_MSG)
        se = pt.split_mo_energy()
        if eris.unrestricted:
            return ukernel(eris.with_df, eris.occ_coeff, eris.vir_coeff, [s[1] for s in se], [s[2] for s in se], with_t2)
        return kernel(eris.with_df, eris.occ_coeff, eris.vir_coeff, se[1], se[2], with_t2)

    pt.ao2mo = _eris_ao2mo(pt, 'DF-MP2 on the GPU')
    pt.init_amps = init_amps
    return pt


def times(with_df):
    """Milliseconds of the last DF-MP2 call: {'stage1', 'stage2'} device time of the half transform and of the pair kernel
    (CUDA events), 'total' host time of the whole call."""
    return _times(with_df, 'b200jk_df_mp2_times', ('stage1', 'stage2', 'total'))
