"""Density-fitted J/K on H100 behind the reference's `with_df` surface.

Mirrors (names, argument meaning, shapes):
  * df.DF(mol, auxbasis): build(), reset(), get_naoaux(), loop(), get_jk(dm, hermi, with_j, with_k,
    direct_scf_tol, omega), range_coulomb(omega), ao2mo = get_mo_eri, get_eri = get_ao_eri
                                                                       pyscf/df/df.py:56-333
  * df_jk.get_jk algebra incl. the mo_coeff/mo_occ fast path           pyscf/df/df_jk.py:280-413
  * addons.make_auxmol / predefined auxiliary basis                    pyscf/df/addons.py:230-361
  * density_fit(mf) installer                                          pyscf/df/df_jk.py:31-107
The three-index tensor is built on the GPU (Rys kernels + cuSOLVER/cuBLAS for the metric) and stays
resident in HBM in the reference layout cderi[naux, nao(nao+1)/2]; the rows of a tensor larger than the GPU that do not fit
live in pinned host memory and are streamed through the GPU once per J/K call (set_device_rows, row_split).
A Cartesian molecule (mol.cart = True) gets a Cartesian tensor [naux_cart, ncart(ncart+1)/2] in a Cartesian auxiliary basis, as
the reference's make_auxmol / cholesky_eri give it (pyscf/df/addons.py:245, pyscf/df/incore.py:144-149).
With pair_tol (opt-in, no reference equivalent) the tensor stores only the AO-pair columns whose Schwarz bound is >= pair_tol
(pair_stats); loop(), cderi_columns(), save() and _cderi still return the reference layout, exact zeros at dropped columns.
"""
import ctypes

import numpy as np

from . import lib as _lib
from .gto.mole import make_auxmol


def _is_cart(mol):
    return bool(getattr(mol, 'cart', False))


def _nao(mol):
    """AO count in the molecule's own convention: (l+1)(l+2)/2 functions per shell when mol.cart, else 2l+1."""
    return int(mol.ao_loc_nr(cart=_is_cart(mol))[-1])


def _check_aux_cart(mol, auxmol):
    """The tensor's auxiliary functions follow the AO convention; a user-assigned auxmol of the other one is refused with the
    reference's messages (pyscf/df/incore.py:144-147)."""
    if not _is_cart(mol) and _is_cart(auxmol):
        raise NotImplementedError('Interface for int3c2e_ssc')
    if _is_cart(mol) and not _is_cart(auxmol):
        raise RuntimeError('Cartesian orbitals for mol and spherical orbitals for auxmol not supported')


def _iden_coeffs(mo1, mo2):
    """ao2mo.incore.iden_coeffs (pyscf/ao2mo/incore.py:239-241): the same object, or equal shapes within 1e-13 (empty sets of
    equal shape count as equal)."""
    if mo1 is mo2:
        return True
    a, b = np.asarray(mo1), np.asarray(mo2)
    return a.shape == b.shape and bool(a.size == 0 or abs(a - b).max() < 1e-13)


# ---- shared by the MO consumers of the tensor (DF.ao2mo, pyscf_b200.dfmp2, pyscf_b200.rpa) ------------------------------------

def _check_df(with_df, method, why):
    """nao of a built, unsharded with_df; method names the caller in the message, why says what sharding would break."""
    if with_df.shard is not None:
        raise NotImplementedError('%s on a sharded tensor (DF(shard=...)) is not implemented: %s' % (method, why))
    with_df.get_naoaux()
    return with_df.nao


def _coeff(c, nao, what, method):
    """c as a contiguous float64 [nao, n] array; complex coefficients and a wrong nao are refused."""
    a = np.asarray(c)
    if np.iscomplexobj(a):
        raise NotImplementedError('%s: complex MO coefficients are not supported' % method)
    if a.ndim != 2 or a.shape[0] != nao:
        raise ValueError('%s: %s coefficients must be [nao, n] with nao = %d, got shape %s' % (method, what, nao, a.shape))
    return np.ascontiguousarray(a, dtype=np.float64)


class _ERIS:
    """What DF-MP2 and DF-RPA need of DFMP2.ao2mo's result (_make_df_eris, pyscf/mp/dfmp2.py:215-272): the active coefficients,
    nocc, nvir, naux.  L[P, ia] stays on the device, so its blocks cannot be read."""

    dtype = np.float64

    def __init__(self, with_df, occ_coeff, vir_coeff, unrestricted, who):
        self.with_df = with_df
        self.occ_coeff, self.vir_coeff = occ_coeff, vir_coeff
        self.unrestricted = unrestricted
        self.naux = with_df.get_naoaux()
        if unrestricted:
            self.nocc = tuple(c.shape[1] for c in occ_coeff)
            self.nvir = tuple(c.shape[1] for c in vir_coeff)
        else:
            self.nocc, self.nvir = occ_coeff.shape[1], vir_coeff.shape[1]
        self._who = who

    def get_ov_blk(self, *args):
        raise NotImplementedError('%s keeps L[P, ia] on the device; get_ov_blk is not available' % self._who)

    def get_occ_blk(self, *args):
        raise NotImplementedError('%s keeps L[P, ia] on the device; get_occ_blk is not available' % self._who)


def _eris_ao2mo(obj, who):
    """The ao2mo(mo_coeff, ovL, ovL_to_save) that patch() puts on a DFMP2 / RPA instance obj: the active orbitals of
    obj.split_mo_coeff() as an _ERIS."""
    def ao2mo(mo_coeff=None, ovL=None, ovL_to_save=None):
        if ovL is not None or ovL_to_save is not None:
            raise NotImplementedError('%s keeps the ovL integrals on the device; ovL / ovL_to_save are not supported' % who)
        sp = obj.split_mo_coeff()
        if len(sp) == 2:
            return _ERIS(obj.with_df, tuple(s[1] for s in sp), tuple(s[2] for s in sp), True, who)
        return _ERIS(obj.with_df, sp[1], sp[2], False, who)
    return ao2mo


def _times(with_df, fn, keys):
    """{key: ms} of the last call, from the C function fn (b200jk_df_*_times)."""
    h = with_df._handle
    ms = np.zeros(len(keys))
    h.check(getattr(h.lib, fn)(h._h, _lib.dptr(ms), len(keys)), fn)
    return dict(zip(keys, ms.tolist()))


class DF:
    def __init__(self, mol, auxbasis=None, device=0, libpath=None, shard=None, pair_tol=None):
        self.mol = mol
        self.auxbasis = auxbasis
        self.auxmol = None
        self.device = device
        self._libpath = libpath
        self.shard = shard         # (rank, world): build only this rank's auxiliary rows (multi-GPU, see parallel.py)
        self._handle = None
        self._vjopt = None         # handle holding only the factorised metric (integral-direct J, get_j)
        self._rsh_df = {}          # omega -> DF (pyscf/df/df.py:298-333 range_coulomb)
        self._cderi_in = None      # tensor assigned by the caller (ndarray or .npy path), used instead of building one
        self.omega = None
        self.lindep = 1e-7         # pyscf/df/incore.py:30-33 LINEAR_DEP_THR
        self.blockdim = 240        # pyscf/df/df.py:95 (loop() default block size)
        self.k_engine = 'tcgen05'
        self.k_slices = 7
        self.device_rows = -1      # cap on the tensor rows kept in HBM, the rest in pinned host memory (-1: automatic)
        # pair screening: keep only the AO-pair columns whose shell-pair Schwarz bound sqrt((ab|ab)) is >= pair_tol (None: dense,
        # the reference's tensor).  A dropped column has 2-norm < pair_tol.  Applies to built tensors, not to an assigned _cderi.
        self.pair_tol = pair_tol
        self.verbose = getattr(mol, 'verbose', 0)
        self.stdout = getattr(mol, 'stdout', None)
        self.max_memory = getattr(mol, 'max_memory', 4000)

    # ---- construction ------------------------------------------------------------------------------
    def build(self):
        mol = self.mol
        if self._cderi_in is not None:
            return self._build_from_cderi()
        if self.auxmol is None:
            self.auxmol = make_auxmol(mol, self.auxbasis)
        aux = self.auxmol
        _check_aux_cart(mol, aux)
        h = _lib.Handle(mol._atm, mol._bas, np.array(mol._env, dtype=np.float64), device=self.device,
                        libpath=self._libpath, cart=_is_cart(mol))
        atm = np.ascontiguousarray(aux._atm, dtype=np.int32)
        bas = np.ascontiguousarray(aux._bas, dtype=np.int32)
        env = np.ascontiguousarray(aux._env, dtype=np.float64)
        omega = self._effective_omega()
        if self.shard is not None:
            h.check(h.lib.b200jk_set_shard(h._h, int(self.shard[0]), int(self.shard[1])), 'b200jk_set_shard')
        self._built_omega = omega
        h.check(h.lib.b200jk_df_set_device_rows(h._h, int(self.device_rows)), 'b200jk_df_set_device_rows')
        h.check(h.lib.b200jk_df_set_pair_tol(h._h, float(self.pair_tol or 0.0)), 'b200jk_df_set_pair_tol')
        h.check(h.lib.b200jk_df_build(h._h, _lib.iptr(atm), len(atm), _lib.iptr(bas), len(bas), _lib.dptr(env), len(env),
                                      omega, self.lindep), 'b200jk_df_build')
        self._handle = h
        self.nao = _nao(mol)
        self.set_k_engine(self.k_engine, self.k_slices)
        return self

    def _effective_omega(self):
        """Operator of the tensor: self.omega when set (range_coulomb children), else what the molecule carries in
        env[PTR_RANGE_OMEGA] — mol.omega or an enclosing `with mol.with_range_coulomb(w)`, as the reference's integral calls see
        it (pyscf/df/incore.py:129-220 runs under the molecule's environment)."""
        if self.omega is not None:
            return float(self.omega)
        return float(self.mol._env[8])

    def _build_from_cderi(self):
        """Upload an assigned tensor (mf.with_df._cderi = ndarray | 'file.npy'; pyscf/df/df.py:116-118,
        pyscf/df/test/test_df_jk.py:135-142) instead of computing 3-center integrals."""
        mol = self.mol
        c = self._cderi_in
        if isinstance(c, str):
            c = np.load(c, mmap_mode='r')
        nao = _nao(mol)
        npair = nao * (nao + 1) // 2
        if c.ndim != 2 or c.shape[1] != npair:
            raise RuntimeError('cderi must have shape (naux, nao*(nao+1)/2) = (*, %d), got %s' % (npair, c.shape))
        c = np.ascontiguousarray(c, dtype=np.float64)
        h = _lib.Handle(mol._atm, mol._bas, np.array(mol._env, dtype=np.float64), device=self.device, libpath=self._libpath,
                        cart=_is_cart(mol))
        if self.shard is not None:
            h.check(h.lib.b200jk_set_shard(h._h, int(self.shard[0]), int(self.shard[1])), 'b200jk_set_shard')
        h.check(h.lib.b200jk_df_set_device_rows(h._h, int(self.device_rows)), 'b200jk_df_set_device_rows')
        h.check(h.lib.b200jk_df_set_cderi(h._h, _lib.dptr(c), c.shape[0], nao), 'b200jk_df_set_cderi')
        self._handle = h
        self.nao = nao
        self.set_k_engine(self.k_engine, self.k_slices)
        return self

    def save(self, path):
        """Write the tensor to `path` (.npy, the reference layout) — the role of DF._cderi_to_save (pyscf/df/df.py:112-118,
        which writes HDF5; h5py is not a dependency here).  Reload with `DF(mol)._cderi = path`."""
        np.save(path, self._cderi)
        return path

    def set_k_engine(self, engine='tcgen05', nslices=7):
        """'tcgen05' (the engine's historical name: int8-slice GEMMs on the tensor cores, wgmma; default) or 'dgemm'
        (cuBLAS FP64 yardstick)."""
        self.k_engine, self.k_slices = engine, nslices
        if self._handle is not None:
            h = self._handle
            h.check(h.lib.b200jk_df_set_kmode(h._h, 1 if engine == 'tcgen05' else 0, nslices), 'b200jk_df_set_kmode')
        return self

    def set_device_rows(self, n=-1):
        """Keep at most `n` rows of this rank's tensor in HBM and the rest in pinned host memory, streamed through the GPU
        once per J/K call (-1: automatic, every row on the device when the tensor fits).  Applied at the next build."""
        self.device_rows = -1 if n is None else int(n)
        return self

    def row_split(self):
        """(rows in HBM, rows in pinned host memory) of this rank's tensor."""
        self.get_naoaux()
        h = self._handle
        n_dev, n_host = ctypes.c_int(0), ctypes.c_int(0)
        h.check(h.lib.b200jk_df_row_split(h._h, ctypes.byref(n_dev), ctypes.byref(n_host)), 'b200jk_df_row_split')
        return n_dev.value, n_host.value

    def pair_stats(self):
        """(kept AO-pair columns, nao(nao+1)/2) of the tensor; equal without pair screening."""
        self.get_naoaux()
        h = self._handle
        ncol, npair = ctypes.c_int64(0), ctypes.c_int64(0)
        h.check(h.lib.b200jk_df_pair_stats(h._h, ctypes.byref(ncol), ctypes.byref(npair)), 'b200jk_df_pair_stats')
        return ncol.value, npair.value

    def stream_stats(self):
        """Host rows streamed by the last get_jk: {'bytes', 'copy_ms', 'exposed_ms'} (exposed: copy time not hidden
        behind compute)."""
        h = self._handle
        b, c, e = ctypes.c_int64(0), ctypes.c_double(0), ctypes.c_double(0)
        h.check(h.lib.b200jk_df_stream_stats(h._h, ctypes.byref(b), ctypes.byref(c), ctypes.byref(e)), 'b200jk_df_stream_stats')
        return {'bytes': b.value, 'copy_ms': c.value, 'exposed_ms': e.value}

    def reset(self, mol=None):
        if mol is not None:
            self.mol = mol
        self.auxmol = None
        if self._handle is not None:
            self._handle.close()
        if getattr(self, '_vjopt', None) is not None:
            self._vjopt.close()
        for child in self._rsh_df.values():
            child.reset()
        self._handle = None
        self._vjopt = None
        self._rsh_df = {}
        self._built_omega = None
        return self

    def get_naoaux(self):
        if self._handle is None:
            self.build()
        n = ctypes.c_int(0)
        h = self._handle
        h.check(h.lib.b200jk_df_naux(h._h, ctypes.byref(n)), 'b200jk_df_naux')
        return n.value

    def loop(self, blksize=None):
        """Yield host copies of cderi row blocks [nrow, nao(nao+1)/2] (pyscf/df/df.py:214-242)."""
        self.get_naoaux()
        row0, naux = ctypes.c_int(0), ctypes.c_int(0)
        self._handle.check(self._handle.lib.b200jk_df_local_rows(self._handle._h, ctypes.byref(row0), ctypes.byref(naux)),
                           'b200jk_df_local_rows')
        naux = naux.value      # rows held by this rank (all of them unless the build was sharded)
        blksize = blksize or self.blockdim
        npair = self.nao * (self.nao + 1) // 2
        h = self._handle
        for r0 in range(0, naux, blksize):
            nr = min(blksize, naux - r0)
            buf = np.empty((nr, npair))
            h.check(h.lib.b200jk_df_get_cderi(h._h, _lib.dptr(buf), r0, nr), 'b200jk_df_get_cderi')
            yield buf

    def cderi_columns(self, cols):
        """cderi[:, cols] for packed AO-pair indices `cols` (mu(mu+1)/2 + nu, mu >= nu), rows held by this rank — numpy slicing
        of the reference's ndarray tensor (pyscf/df/df.py:116) without copying the tensor to the host."""
        self.get_naoaux()
        h = self._handle
        row0, nrow = ctypes.c_int(0), ctypes.c_int(0)
        h.check(h.lib.b200jk_df_local_rows(h._h, ctypes.byref(row0), ctypes.byref(nrow)), 'b200jk_df_local_rows')
        cols = np.ascontiguousarray(cols, dtype=np.int64)
        out = np.empty((nrow.value, len(cols)))
        h.check(h.lib.b200jk_df_get_cderi_cols(h._h, _lib.dptr(out), cols.ctypes.data_as(ctypes.POINTER(ctypes.c_int64)), len(cols)),
                'b200jk_df_get_cderi_cols')
        return out

    @property
    def _cderi(self):
        return np.vstack(list(self.loop()))

    @_cderi.setter
    def _cderi(self, value):
        # assigning a tensor discards whatever was built (reset() keeps the assignment, like the reference keeps _cderi)
        if self._handle is not None:
            self._handle.close()
            self._handle = None
        self._cderi_in = value

    def range_coulomb(self, omega):
        key = float(omega)
        if key not in self._rsh_df:
            rsh = DF(self.mol, self.auxbasis, device=self.device, libpath=self._libpath, shard=self.shard)
            rsh.auxmol = self.auxmol
            rsh.omega = key
            rsh.lindep = self.lindep
            rsh.k_engine, rsh.k_slices = self.k_engine, self.k_slices
            rsh.device_rows = self.device_rows
            rsh.pair_tol = self.pair_tol       # screened with the bound of its own operator
            self._rsh_df[key] = rsh.build()
        return self._rsh_df[key]

    # ---- J/K -----------------------------------------------------------------------------------------
    def _prepare_j(self):
        """Auxiliary tables + factorised metric only (the reference's cached dfobj._vjopt, df_jk.py:422-455)."""
        mol = self.mol
        if self.auxmol is None:
            self.auxmol = make_auxmol(mol, self.auxbasis)
        aux = self.auxmol
        _check_aux_cart(mol, aux)
        h = _lib.Handle(mol._atm, mol._bas, np.array(mol._env, dtype=np.float64), device=self.device,
                        libpath=self._libpath, cart=_is_cart(mol))
        atm = np.ascontiguousarray(aux._atm, dtype=np.int32)
        bas = np.ascontiguousarray(aux._bas, dtype=np.int32)
        env = np.ascontiguousarray(aux._env, dtype=np.float64)
        omega = self._effective_omega()
        self._built_omega = omega
        h.check(h.lib.b200jk_df_prepare_j(h._h, _lib.iptr(atm), len(atm), _lib.iptr(bas), len(bas), _lib.dptr(env),
                                          len(env), omega, self.lindep), 'b200jk_df_prepare_j')
        self._vjopt = h
        self.nao = _nao(mol)
        return h

    def get_j(self, dm, hermi=0, direct_scf_tol=1e-13):
        """Integral-direct J without the three-index tensor: rho = j2c^-1 (P|ij) D_ji, J_ij = (ij|P) rho_P, two passes
        over the 3-center integrals on the GPU (df_jk.get_j, pyscf/df/df_jk.py:415-506)."""
        if self._cderi_in is not None:     # an assigned tensor has no auxiliary basis / metric attached: J from the tensor
            return self.get_jk(dm, hermi, True, False, direct_scf_tol)[0]
        h = self._handle or getattr(self, '_vjopt', None) or self._prepare_j()
        nao = self.nao
        dm = np.asarray(dm)
        if dm.shape[-1] != nao or dm.shape[-2] != nao:
            raise RuntimeError('dm shape %s does not match nao=%d' % (dm.shape, nao))
        if np.iscomplexobj(dm):
            return self.get_j(dm.real, hermi, direct_scf_tol) + 1j * self.get_j(dm.imag, hermi, direct_scf_tol)
        shape = dm.shape
        dms = np.ascontiguousarray(dm.reshape(-1, nao, nao), dtype=np.float64)
        vj = np.empty_like(dms)
        h.check(h.lib.b200jk_df_direct_j(h._h, _lib.dptr(dms), len(dms), nao, _lib.dptr(vj)), 'b200jk_df_direct_j')
        return vj.reshape(shape)

    def get_jk(self, dm, hermi=1, with_j=True, with_k=True, direct_scf_tol=1e-13, omega=None):
        if omega is not None and float(omega) != self._effective_omega():
            # pyscf/df/df.py:259-296: a different operator lives on its own cached DF object (omega = 0: the plain Coulomb one)
            return self.range_coulomb(omega).get_jk(dm, hermi, with_j, with_k, direct_scf_tol)
        if self._cderi_in is None and (self._handle is not None or self._vjopt is not None) and \
                getattr(self, '_built_omega', None) not in (None, self._effective_omega()):
            self.reset()       # the molecule's own operator changed since the tensor was built (mol.omega, with_range_coulomb)
        if not with_k and self._handle is None and self.shard is None and self._cderi_in is None:
            # J only and no tensor yet: integral-direct J (pyscf/df/df_jk.py:282-285)
            return self.get_j(dm, hermi, direct_scf_tol), None
        if self._handle is None:
            self.build()
        mo_coeff = getattr(dm, 'mo_coeff', None)
        mo_occ = getattr(dm, 'mo_occ', None)
        dm = np.asarray(dm)
        nao = self.nao
        if dm.shape[-1] != nao or dm.shape[-2] != nao:
            raise RuntimeError('dm shape %s does not match nao=%d' % (dm.shape, nao))
        if np.iscomplexobj(dm):
            vjr, vkr = self.get_jk(dm.real, 0, with_j, with_k)
            vji, vki = self.get_jk(dm.imag, 0, with_j, with_k)
            return (None if vjr is None else vjr + 1j * vji), (None if vkr is None else vkr + 1j * vki)
        shape = dm.shape
        dms = np.ascontiguousarray(dm.reshape(-1, nao, nao), dtype=np.float64)
        n_dm = len(dms)
        h = self._handle
        vj = np.empty_like(dms) if with_j else None
        vk = np.empty_like(dms) if with_k else None
        # fast K path when the density carries its orbitals (pyscf/df/df_jk.py:339-357): one orbital set per density
        # matrix; an ROHF-style tag (half as many orbital sets as densities) is expanded into (occupied, doubly occupied)
        orbo = None
        if with_k and mo_coeff is not None and mo_occ is not None:
            mo_occ = np.asarray(mo_occ, dtype=np.float64)
            nmo = mo_occ.shape[-1]
            mo_coeff = np.asarray(mo_coeff, dtype=np.float64).reshape(-1, nao, nmo)
            mo_occ = mo_occ.reshape(-1, nmo)
            if mo_occ.shape[0] * 2 == n_dm and len(mo_coeff) * 2 == n_dm:          # ROHF density pair (df_jk.py:346-351)
                mo_coeff = np.vstack((mo_coeff, mo_coeff))
                occa = (mo_occ > 0).astype(np.float64)
                occb = (mo_occ == 2).astype(np.float64)
                if occa.sum() + occb.sum() != mo_occ.sum():
                    raise RuntimeError('ROHF-style mo_occ must hold occupations 0, 1, 2')
                mo_occ = np.vstack((occa, occb))
            if len(mo_coeff) == n_dm and mo_occ.shape[0] == n_dm and (mo_occ >= 0).all():
                orbo = [np.ascontiguousarray(mo_coeff[k][:, mo_occ[k] > 0] * np.sqrt(mo_occ[k][mo_occ[k] > 0])) for k in range(n_dm)]
        if orbo is None or n_dm == 1:
            occ = None if orbo is None else orbo[0][None]
            nocc = 0 if orbo is None else orbo[0].shape[1]
            if orbo is not None and nocc == 0:
                occ = None      # no occupied orbital: K = 0 through the general path
            h.check(h.lib.b200jk_df_jk(h._h, _lib.dptr(dms), n_dm, nao, _lib.dptr(occ), nocc, int(hermi), _lib.dptr(vj),
                                       _lib.dptr(vk)), 'b200jk_df_jk')
        else:
            # several orbital sets (UHF, ROHF, state-averaged): J for all densities in one pass over the tensor, K set by set
            # through the single-set occupied-orbital call (the tensor-core engine)
            if with_j:
                h.check(h.lib.b200jk_df_jk(h._h, _lib.dptr(dms), n_dm, nao, None, 0, int(hermi), _lib.dptr(vj), None), 'b200jk_df_jk')
            for k in range(n_dm):
                nocc = orbo[k].shape[1]
                if nocc == 0:
                    vk[k] = 0.0
                    continue
                h.check(h.lib.b200jk_df_jk(h._h, _lib.dptr(dms[k:k + 1]), 1, nao, _lib.dptr(orbo[k][None]), nocc, int(hermi), None,
                                           _lib.dptr(vk[k:k + 1])), 'b200jk_df_jk')
        return (None if vj is None else vj.reshape(shape)), (None if vk is None else vk.reshape(shape))

    # ---- MO / AO integrals from the tensor ------------------------------------------------------------
    def ao2mo(self, mo_coeffs, compact=True):
        """(ij|kl) = sum_P L[P, ij] L[P, kl], L[P, ij] = C1[:, i]^T B_P C2[:, j], on the GPU: DF.ao2mo (pyscf/df/df.py:278-296),
        what DF-CASSCF and DF-NEVPT2 call on mf.with_df (DF-MP2 takes its own route: pyscf_b200.dfmp2).

        mo_coeffs: one [nao, n] array (four equal sets) or a sequence of four.  Pair (1,2) is packed s2 (row i(i+1)/2 + j,
        i >= j) when `compact` and its two sets are identical in the sense of iden_coeffs (pyscf/ao2mo/incore.py:239-241),
        else s1 (row i n2 + j); pair (3,4) alike.  Returns [nij, nkl] float64."""
        if self.shard is not None:
            raise NotImplementedError('DF.ao2mo on a sharded tensor (DF(shard=...)) is not implemented')
        if isinstance(mo_coeffs, np.ndarray) and mo_coeffs.ndim == 2:
            mo_coeffs = (mo_coeffs,) * 4
        if len(mo_coeffs) != 4:
            raise ValueError('DF.ao2mo needs one [nao, n] array or four of them, got %d' % len(mo_coeffs))
        self.get_naoaux()
        mo_coeffs = [np.asarray(c) for c in mo_coeffs]
        cs = [_coeff(c, self.nao, 'MO', 'DF.ao2mo') for c in mo_coeffs]
        # _conc_mos (pyscf/ao2mo/incore.py:244-262): s2 only for identical sets given in double precision
        s12 = bool(compact) and np.result_type(*mo_coeffs[:2]) == np.double and _iden_coeffs(mo_coeffs[0], mo_coeffs[1])
        s34 = bool(compact) and np.result_type(*mo_coeffs[2:]) == np.double and _iden_coeffs(mo_coeffs[2], mo_coeffs[3])
        sym = s12 == s34 and _iden_coeffs(mo_coeffs[0], mo_coeffs[2]) and _iden_coeffs(mo_coeffs[1], mo_coeffs[3])
        n = [a.shape[1] for a in cs]
        nij = n[0] * (n[0] + 1) // 2 if s12 else n[0] * n[1]
        nkl = n[2] * (n[2] + 1) // 2 if s34 else n[2] * n[3]
        out = np.empty((nij, nkl))
        if out.size == 0:
            return out
        h = self._handle
        if sym:
            h.check(h.lib.b200jk_df_ao2mo(h._h, _lib.dptr(cs[0]), n[0], _lib.dptr(cs[1]), n[1], int(s12), None, 0, None, 0, 0,
                                          _lib.dptr(out)), 'b200jk_df_ao2mo')
        else:
            h.check(h.lib.b200jk_df_ao2mo(h._h, _lib.dptr(cs[0]), n[0], _lib.dptr(cs[1]), n[1], int(s12), _lib.dptr(cs[2]), n[2],
                                          _lib.dptr(cs[3]), n[3], int(s34), _lib.dptr(out)), 'b200jk_df_ao2mo')
        return out
    get_mo_eri = ao2mo

    def get_eri(self):
        """ao2mo.restore(8, sum_P B[P]^T B[P], nao) on the GPU (DF.get_eri, pyscf/df/df.py:269-276): the lower triangle, row by
        row, of the [npair, npair] AO-pair matrix (npair = nao(nao+1)/2), a vector of npair(npair+1)/2."""
        if self.shard is not None:
            raise NotImplementedError('DF.get_eri on a sharded tensor (DF(shard=...)) is not implemented')
        self.get_naoaux()
        npair = self.nao * (self.nao + 1) // 2
        out = np.empty(npair * (npair + 1) // 2)
        h = self._handle
        h.check(h.lib.b200jk_df_get_ao_eri(h._h, _lib.dptr(out)), 'b200jk_df_get_ao_eri')
        return out
    get_ao_eri = get_eri

    def ao2mo_times(self):
        """Milliseconds of the last ao2mo / get_eri: {'stage1', 'stage2'} device time of the half transforms and of the
        output GEMMs (CUDA events), 'total' host time of the whole call including the copies to the caller."""
        return _times(self, 'b200jk_df_ao2mo_times', ('stage1', 'stage2', 'total'))

    def stats(self):
        return self._handle.stats()

    def stage_times(self):
        """Device time per stage of the last get_jk: {'j_rho' | 'j_acc' | 'k_gemm1' | 'k_slice' | 'k_gemm2': (ms, launches)}."""
        return self._handle.df_stage_times()


class TaggedDM(np.ndarray):
    """ndarray carrying mo_coeff / mo_occ like lib.tag_array (pyscf/lib/numpy_helper.py:1460-1500; hf.py:868).

    As in the reference the tags describe THIS array's contents only: any ufunc result (dm - dm_last, 0.5 * dm, ...) comes
    back as a plain ndarray (`__array_wrap__`, numpy_helper.py:1477-1484) and views / slices start without tags, so a derived
    density can never reach the occupied-orbital K path with stale orbitals."""
    mo_coeff = None
    mo_occ = None

    def __new__(cls, a, mo_coeff=None, mo_occ=None):
        obj = np.asarray(a).view(cls)
        obj.mo_coeff = mo_coeff
        obj.mo_occ = mo_occ
        return obj

    def __array_wrap__(self, out, context=None, return_scalar=False):
        if out.ndim == 0:
            return out[()]
        return out.view(np.ndarray)

    def __reduce__(self):
        pickled = np.ndarray.__reduce__(self)
        return (pickled[0], pickled[1], pickled[2] + ((self.mo_coeff, self.mo_occ),))

    def __setstate__(self, state):
        np.ndarray.__setstate__(self, state[:-1])
        self.mo_coeff, self.mo_occ = state[-1]


def tag_array(a, **kwargs):
    """lib.tag_array (pyscf/lib/numpy_helper.py:1487-1500)."""
    t = TaggedDM(a, getattr(a, 'mo_coeff', None), getattr(a, 'mo_occ', None))
    for k, v in kwargs.items():
        setattr(t, k, v)
    return t


class _DFHF:
    """Mixin placed in front of the mean-field class by density_fit(), the role of df_jk._DFHF (pyscf/df/df_jk.py:104-179):
    get_jk goes to with_df; only_dfj routes K to the exact 4-center builder; direct_scf := only_dfj; reset() resets with_df."""
    only_dfj = None

    def reset(self, mol=None):
        if self.with_df is not None:
            self.with_df.reset(mol)
        vh = getattr(self, '_b200_direct_jk', None)
        if vh is not None and hasattr(vh, '_cache'):
            vh._cache.clear()
        return super().reset(mol)

    def get_jk(self, mol=None, dm=None, hermi=1, with_j=True, with_k=True, omega=None):
        assert with_j or with_k
        if mol is None:
            mol = self.mol
        if dm is None:
            dm = self.make_rdm1()
        if not self.with_df:       # mf.with_df = None switches density fitting off (df_jk.py:153-154)
            return self._exact_get_jk(mol, dm, hermi, with_j, with_k, omega)
        vj = vk = None
        with_dfk = with_k and not self.only_dfj
        if with_j or with_dfk:
            vj, vk = self.with_df.get_jk(dm, hermi, with_j, with_dfk, getattr(self, 'direct_scf_tol', 1e-13), omega)
        if with_k and not with_dfk:
            vk = self._exact_get_jk(mol, dm, hermi, False, True, omega)[1]
        return vj, vk

    def _exact_get_jk(self, mol, dm, hermi, with_j, with_k, omega):
        """super().get_jk of the reference: the GPU 4-center builder when jk.patch() was applied to the object before (its
        instance override is kept as _b200_direct_jk), else the mean-field class's own get_jk."""
        f = getattr(self, '_b200_direct_jk', None)
        if f is not None:
            return f(mol, dm, hermi, with_j, with_k, omega)
        return super().get_jk(mol, dm, hermi, with_j, with_k, omega)


def density_fit(mf, auxbasis=None, with_df=None, only_dfj=False, device=0):
    """df_jk.density_fit (pyscf/df/df_jk.py:31-102) with a GPU DF object: returns an object of the dynamic class
    (_DFHF, mf.__class__) sharing mf's attributes, whose get_jk is served by with_df.get_jk (J and K from the fitted tensor) or,
    with only_dfj=True, J from the tensor and K from the exact 4-center path (RIJONX, df_jk.py:157-179).  An object that is
    already density-fitted just gets the new with_df / only_dfj (df_jk.py:88-99)."""
    if with_df is None:
        with_df = DF(mf.mol, auxbasis, device=device)
        with_df.verbose = getattr(mf, 'verbose', 0)
        with_df.stdout = getattr(mf, 'stdout', None)
        with_df.max_memory = getattr(mf, 'max_memory', 4000)
    if isinstance(mf, _DFHF):
        mf.with_df = with_df
        mf.only_dfj = only_dfj
        mf.direct_scf = only_dfj
        return mf
    base = mf.__class__
    cls = type('DF' + base.__name__, (_DFHF, base), {})
    dfmf = object.__new__(cls)
    dfmf.__dict__.update(mf.__dict__)
    # an instance-level get_jk (jk.patch) would shadow the class method: keep it as the exact builder instead
    inst = dfmf.__dict__.pop('get_jk', None)
    if inst is not None:
        dfmf._b200_direct_jk = inst
    dfmf.__dict__.pop('reset', None)      # jk.patch's reset wrapper: _DFHF.reset clears the same cache
    if inst is not None and getattr(mf, '_b200_opts', None) is not None:
        inst._cache = mf._b200_opts
    dfmf._eri = None
    dfmf.with_df = with_df
    dfmf.only_dfj = only_dfj
    dfmf.direct_scf = only_dfj     # df_jk.py:133-137: incremental direct-SCF K only when K is the exact one
    return dfmf


def get_jk_only_dfj(with_df, mol, dm, hermi=1, with_j=True, with_k=True, omega=None, direct_scf_tol=1e-13, vhfopt=None):
    """_DFHF.get_jk with only_dfj=True (pyscf/df/df_jk.py:157-179): vj from the DF object, vk from the exact
    4-center path of jk.get_jk."""
    from . import jk as _jk
    vj = vk = None
    if with_j:
        vj = with_df.get_jk(dm, hermi, True, False, direct_scf_tol, omega)[0]
    if with_k:
        vk = _jk.get_jk(mol, dm, hermi, vhfopt, False, True, omega)[1]
    return vj, vk
