"""Direct RPA on the GPU from the resident density-fitting tensor: the RPA / URPA kernels of pyscf/gw/rpa.py:43-145 and
pyscf/gw/urpa.py:41-72 without the tensor or L[P, ia] ever reaching the host.

  * kernel(with_df, occ_coeffs, vir_coeffs, e_ovs, f_ovs, nw=40, x0=0.5)     e_corr = sum_w weight / 2pi (log det(I - Pi(w))
                                                                              + tr Pi(w)) on the scaled Gauss-Legendre grid
  * kernel_terms(with_df, occ_coeffs, vir_coeffs, e_ovs, f_ovs, omegas)      (log det(I - Pi(w)), tr Pi(w)) per frequency
  * dielectric_matrix(with_df, occ_coeffs, vir_coeffs, e_ovs, f_ovs, omega)  Pi(omega) [naux, naux]
  * patch(rpa)   route a PySCF RPA / URPA instance whose with_df is a pyscf_b200.df.DF through the kernels above
  * times(with_df)

occ_coeffs / vir_coeffs / e_ovs / f_ovs: one spin (an [nao, n] array, a 1-D [nocc nvir] array) or a sequence of two (URPA).
Pi(w) = sum_s L_s chi_s(w) L_s^T with chi_s[ia] = 2 e_ov f_ov / (w^2 + e_ov^2) is formed on the device one frequency at a time,
and log det(I - Pi) is taken from its Cholesky factor (b200jk_df_rpa, df_rpa.cuh).  The reference's np.log(np.linalg.det(.))
overflows once the log-determinant passes ~709; the Cholesky form agrees with it wherever it is finite.  This module does not
import pyscf: patch() only replaces three methods of the instance it is given.
"""
import numpy as np

from . import lib as _lib
from .df import DF, _check_df, _coeff, _eris_ao2mo, _times

_METHOD = 'DF-RPA'


def scaled_legendre_roots(nw, x0=0.5):
    """_get_scaled_legendre_roots (rpa.py:132-145): the nw Gauss-Legendre roots mapped from [-1, 1] to [0, inf)."""
    freqs, wts = np.polynomial.legendre.leggauss(nw)
    freqs_new = x0 * (1.0 + freqs) / (1.0 - freqs)
    wts = wts * 2.0 * x0 / (1.0 - freqs) ** 2
    return freqs_new, wts


def _spins(x, ndim):
    """One spin given as an array of `ndim` dimensions, or a sequence of per-spin arrays."""
    if isinstance(x, np.ndarray) and x.ndim == ndim:
        return [x]
    return list(x)


def _ov(x, n, what):
    a = np.asarray(x)
    if np.iscomplexobj(a):
        raise NotImplementedError('%s: complex %s is not supported' % (_METHOD, what))
    a = np.ascontiguousarray(a, dtype=np.float64).ravel()
    if len(a) != n:
        raise ValueError('%s: %s has %d entries for nocc * nvir = %d' % (_METHOD, what, len(a), n))
    return a


def _run(with_df, occ_coeffs, vir_coeffs, e_ovs, f_ovs, omegas, with_diel):
    """b200jk_df_rpa: (logdet[nw], trace[nw], Pi or None)."""
    nao = _check_df(with_df, _METHOD, 'Pi needs every auxiliary row of L')
    cos = [_coeff(c, nao, 'occupied', _METHOD) for c in _spins(occ_coeffs, 2)]
    cvs = [_coeff(c, nao, 'virtual', _METHOD) for c in _spins(vir_coeffs, 2)]
    eos, fos = _spins(e_ovs, 1), _spins(f_ovs, 1)
    ns = len(cos)
    if ns not in (1, 2) or len(cvs) != ns or len(eos) != ns or len(fos) != ns:
        raise ValueError('%s: one or two spins of occupied / virtual coefficients, e_ov and f_ov, got %d, %d, %d, %d'
                         % (_METHOD, len(cos), len(cvs), len(eos), len(fos)))
    nocc = np.array([c.shape[1] for c in cos], dtype=np.int32)
    nvir = np.array([c.shape[1] for c in cvs], dtype=np.int32)
    eos = [_ov(e, int(no) * int(nv), 'e_ov') for e, no, nv in zip(eos, nocc, nvir)]
    fos = [_ov(f, int(no) * int(nv), 'f_ov') for f, no, nv in zip(fos, nocc, nvir)]
    omegas = np.ascontiguousarray(np.atleast_1d(np.asarray(omegas, dtype=np.float64)))
    nw = len(omegas)
    logdet, trace = np.zeros(nw), np.zeros(nw)
    naux = with_df.get_naoaux()
    diel = np.zeros((naux, naux)) if with_diel else None
    arr = _lib.c_double_p * ns
    h = with_df._handle
    h.check(h.lib.b200jk_df_rpa(h._h, ns, arr(*[_lib.dptr(c) for c in cos]), _lib.iptr(nocc), arr(*[_lib.dptr(c) for c in cvs]),
                                _lib.iptr(nvir), arr(*[_lib.dptr(x) for x in eos]), arr(*[_lib.dptr(x) for x in fos]), nw,
                                _lib.dptr(omegas), _lib.dptr(logdet), _lib.dptr(trace),
                                _lib.dptr(diel) if with_diel else None), 'b200jk_df_rpa')
    return logdet, trace, diel


def kernel(with_df, occ_coeffs, vir_coeffs, e_ovs, f_ovs, nw=40, x0=0.5):
    """Direct-RPA correlation energy (rpa.kernel, rpa.py:77-92): e_corr = sum_w weight / 2pi (log det(I - Pi(w)) + tr Pi(w))
    over the nw scaled Gauss-Legendre frequencies, summed on the host in frequency order."""
    freqs, wts = scaled_legendre_roots(nw, x0)
    logdet, trace, _ = _run(with_df, occ_coeffs, vir_coeffs, e_ovs, f_ovs, freqs, False)
    e_corr = 0.0
    for weigh, ld, tr in zip(wts, logdet, trace):
        factor = weigh / (2.0 * np.pi)
        e_corr += factor * ld
        e_corr += factor * tr
    return float(e_corr)


def kernel_terms(with_df, occ_coeffs, vir_coeffs, e_ovs, f_ovs, omegas):
    """Per frequency: (log det(I - Pi(w)), tr Pi(w)) as two arrays."""
    logdet, trace, _ = _run(with_df, occ_coeffs, vir_coeffs, e_ovs, f_ovs, omegas, False)
    return logdet, trace


def dielectric_matrix(with_df, occ_coeffs, vir_coeffs, e_ovs, f_ovs, omega):
    """make_dielectric_matrix (rpa.py:100-130, urpa.py:41-72): Pi(omega) = sum_s L_s chi_s L_s^T [naux, naux]."""
    return _run(with_df, occ_coeffs, vir_coeffs, e_ovs, f_ovs, [float(omega)], True)[2]


def patch(rpa):
    """Route a PySCF RPA / URPA instance whose with_df is a pyscf_b200.df.DF through the GPU kernels: rpa.ao2mo,
    rpa.make_dielectric_matrix and rpa.kernel are replaced on the instance.  kernel keeps the reference's sequence (rpa.py:188-210):
    the complex-orbital NotImplementedError, dump_flags, get_e_hf, make_e_ov / make_f_ov (frozen orbitals and the small-gap
    warning stay PySCF's), then e_hf, e_corr and _finalize.  RPA(mf) on an unfitted mf makes a CPU df.DF: set rpa.with_df to a
    pyscf_b200.df.DF first.  Returns rpa."""
    if not isinstance(getattr(rpa, 'with_df', None), DF):
        raise TypeError('%s: rpa.with_df must be a pyscf_b200.df.DF (got %s); set rpa.with_df = pyscf_b200.df.DF(mol, auxbasis)'
                        '.build() before patch()' % (_METHOD, type(getattr(rpa, 'with_df', None)).__name__))

    def make_dielectric_matrix(omega, e_ov=None, f_ov=None, eris=None, max_memory=None, blksize=None):
        if e_ov is None:
            e_ov = rpa.make_e_ov()
        if f_ov is None:
            f_ov = rpa.make_f_ov()
        if eris is None:
            eris = rpa.ao2mo()
        return dielectric_matrix(eris.with_df, eris.occ_coeff, eris.vir_coeff, e_ov, f_ov, omega)

    def kernel_(eris=None, nw=40, x0=0.5):
        if np.iscomplexobj(rpa.mo_coeff):
            raise NotImplementedError
        rpa.dump_flags()
        if eris is None:
            eris = rpa.ao2mo()
        e_hf = rpa.get_e_hf()
        e_ov = rpa.make_e_ov()
        f_ov = rpa.make_f_ov()
        e_corr = kernel(eris.with_df, eris.occ_coeff, eris.vir_coeff, e_ov, f_ov, nw, x0)
        rpa.e_hf, rpa.e_corr = e_hf, e_corr
        rpa._finalize()
        return rpa.e_corr

    rpa.ao2mo = _eris_ao2mo(rpa, _METHOD)
    rpa.make_dielectric_matrix = make_dielectric_matrix
    rpa.kernel = kernel_
    return rpa


def times(with_df):
    """Milliseconds of the last RPA call: {'stage1', 'pi', 'factor'} device time of the half transform, of the Pi GEMMs and of
    the factorisations (CUDA events, summed over the frequencies), 'total' host time of the whole call."""
    return _times(with_df, 'b200jk_df_rpa_times', ('stage1', 'pi', 'factor', 'total'))
