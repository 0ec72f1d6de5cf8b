"""Direct-SCF J/K on H100 behind the reference's plugin surface.

Mirrors (same names, argument meaning, shapes and error behaviour):
  * scf.hf.get_jk(mol, dm, hermi, vhfopt, with_j, with_k, omega)      pyscf/scf/hf.py:963-1034
  * scf.hf.SCF.get_jk / get_j / get_k                                  pyscf/scf/hf.py:2136-2170
  * scf._vhf._VHFOpt (cached screening state, keyed by omega)          pyscf/scf/_vhf.py:151-275;
    SCF._opt dict                                                      pyscf/scf/hf.py:1803,2141-2146
Install on a PySCF mean-field object with `patch(mf)` (instance override of get_jk, the hook
documented in examples/scf/43-custom_get_jk.py:36-45).
"""
import hashlib
import weakref

import numpy as np

from . import lib as _lib

PTR_RANGE_OMEGA = 8      # pyscf/gto/mole.py:80


def effective_omega(mol, omega):
    """The operator a call with `omega` sees (pyscf/scf/hf.py:1021 `with mol.with_range_coulomb(omega)`, pyscf/gto/mole.py:2940-2951,
    3049-3063): an explicit omega wins; None means whatever the molecule already carries in env[PTR_RANGE_OMEGA] (mol.omega or an
    enclosing `with mol.with_range_coulomb(w)`)."""
    if omega is None:
        return float(mol._env[PTR_RANGE_OMEGA])
    return float(omega)


def mol_fingerprint(mol):
    """Identity of the integral tables (geometry, basis): cached optimizers are only reused for identical _atm/_bas/_env
    (everything but the range-separation slot, which is part of the cache key)."""
    env = np.array(mol._env, dtype=np.float64, copy=True)
    env[PTR_RANGE_OMEGA] = 0.0
    hsh = hashlib.sha1()
    hsh.update(np.ascontiguousarray(mol._atm, dtype=np.int32).tobytes())
    hsh.update(np.ascontiguousarray(mol._bas, dtype=np.int32).tobytes())
    hsh.update(env.tobytes())
    hsh.update(b'cart' if getattr(mol, 'cart', False) else b'sph')
    return hsh.hexdigest()


class VHFOpt:
    """Device-resident shell-pair data + Schwarz bounds for one (mol, omega); cf. _vhf._VHFOpt."""

    def __init__(self, mol, direct_scf_tol=1e-13, omega=None, device=0, libpath=None):
        self.mol = mol
        self.direct_scf_tol = direct_scf_tol
        self.omega = effective_omega(mol, omega)
        self.fingerprint = mol_fingerprint(mol)
        self.cart = bool(getattr(mol, 'cart', False))       # Cartesian AOs: libcint's int2e_cart functions (pyscf/gto/mole.py cart=True)
        env = np.array(mol._env, dtype=np.float64, copy=True)
        self.handle = _lib.Handle(mol._atm, mol._bas, env, device=device, libpath=libpath, cart=self.cart)
        self.nao = int(mol.ao_loc_nr(cart=self.cart)[-1]) if hasattr(mol, 'ao_loc_nr') else mol.nao
        h = self.handle
        h.check(h.lib.b200jk_set_screening(h._h, direct_scf_tol, self.omega), 'b200jk_set_screening')

    @property
    def q_cond(self):
        h = self.handle
        nbas = len(h.bas)
        q = np.empty((nbas, nbas))
        h.check(h.lib.b200jk_get_q_cond(h._h, _lib.dptr(q), nbas), 'b200jk_get_q_cond')
        return q

    def get_jk(self, dm, hermi=1, with_j=True, with_k=True):
        dm = np.asarray(dm)
        if np.iscomplexobj(dm):
            # pyscf/scf/hf.py:1017-1031: real and imaginary parts are contracted separately, without symmetry
            vjr, vkr = self.get_jk(dm.real, 0, with_j, with_k)
            vji, vki = self.get_jk(dm.imag, 0, with_j, with_k)
            vj = None if vjr is None else vjr + 1j * vji
            vk = None if vkr is None else vkr + 1j * vki
            return vj, vk
        nao = self.nao
        if dm.shape[-1] != nao or dm.shape[-2] != nao:
            raise RuntimeError('dm shape %s does not match nao=%d' % (dm.shape, nao))
        shape = dm.shape
        dms = np.ascontiguousarray(dm.reshape(-1, nao, nao), dtype=np.float64)
        n_dm = len(dms)
        vj = np.empty_like(dms) if with_j else None
        vk = np.empty_like(dms) if with_k else None
        h = self.handle
        h.check(h.lib.b200jk_direct_jk(h._h, _lib.dptr(dms), n_dm, nao, int(hermi), _lib.dptr(vj), _lib.dptr(vk)),
                'b200jk_direct_jk')
        if vj is not None:
            vj = vj.reshape(shape)
        if vk is not None:
            vk = vk.reshape(shape)
        return vj, vk

    def stats(self):
        return self.handle.stats()

    def close(self):
        self.handle.close()


class _OptCache:
    """Optimizers per (molecule tables, effective omega), like SCF._opt[omega] (pyscf/scf/hf.py:1803,2141-2146).  Entries hang on
    the molecule OBJECT through a weak reference (a dead molecule frees its GPU handles; a recycled id() can never hit a stale
    entry) and are validated against a fingerprint of _atm/_bas/_env, so an in-place mol.build() / set_geom_() gets a fresh one."""

    def __init__(self, max_entries=8):
        self.max_entries = max_entries
        self._d = {}     # id(mol) -> (weakref | None, {omega: VHFOpt})

    def _drop(self, key):
        ent = self._d.pop(key, None)
        if ent:
            for o in ent[1].values():
                o.close()

    def get(self, mol, omega, **kw):
        key = id(mol)
        ent = self._d.get(key)
        if ent is not None and ent[0] is not None and ent[0]() is not mol:
            self._drop(key)
            ent = None
        if ent is None:
            try:
                ref = weakref.ref(mol, lambda _r, k=key: self._drop(k))
            except TypeError:
                ref = None
            while len(self._d) >= self.max_entries:
                self._drop(next(iter(self._d)))
            ent = self._d[key] = (ref, {})
        om = effective_omega(mol, omega)
        opt = ent[1].get(om)
        if opt is not None and (opt.fingerprint != mol_fingerprint(mol) or (ent[0] is None and opt.mol is not mol)):
            opt.close()
            opt = None
        if opt is None:
            opt = ent[1][om] = VHFOpt(mol, omega=omega, **kw)
        return opt

    def clear(self):
        for key in list(self._d):
            self._drop(key)

    def __len__(self):
        return sum(len(ent[1]) for ent in self._d.values())


_opt_cache = _OptCache()


class IncoreJK:
    """J/K from stored two-electron integrals (mf._eri): the role of _vhf.incore / dot_eri_dm (pyscf/scf/_vhf.py:283-366,
    pyscf/scf/hf.py:902-961).  eri: 8-fold packed (mol.intor('int2e', aosym='s8')), 4-fold [npair, npair] or full [nao]^4;
    copied to the device once."""

    def __init__(self, mol, eri, device=0, libpath=None):
        env = np.array(mol._env, dtype=np.float64, copy=True)
        cart = bool(getattr(mol, 'cart', False))
        self.handle = _lib.Handle(mol._atm, mol._bas, env, device=device, libpath=libpath, cart=cart)
        self.nao = int(mol.ao_loc_nr(cart=cart)[-1]) if hasattr(mol, 'ao_loc_nr') else mol.nao
        eri = np.ascontiguousarray(eri, dtype=np.float64)
        self._eri_id = id(eri)
        h = self.handle
        h.check(h.lib.b200jk_incore_set_eri(h._h, _lib.dptr(eri.reshape(-1)), eri.size, self.nao), 'b200jk_incore_set_eri')

    def get_jk(self, dm, hermi=1, with_j=True, with_k=True):
        dm = np.asarray(dm)
        if np.iscomplexobj(dm):
            vjr, vkr = self.get_jk(dm.real, 0, with_j, with_k)
            vji, vki = self.get_jk(dm.imag, 0, with_j, with_k)
            return (None if vjr is None else vjr + 1j * vji), (None if vkr is None else vkr + 1j * vki)
        nao = self.nao
        if dm.shape[-1] != nao or dm.shape[-2] != nao:
            raise RuntimeError('dm shape %s does not match nao=%d' % (dm.shape, nao))
        shape = dm.shape
        dms = np.ascontiguousarray(dm.reshape(-1, nao, nao), dtype=np.float64)
        vj = np.empty_like(dms) if with_j else None
        vk = np.empty_like(dms) if with_k else None
        h = self.handle
        h.check(h.lib.b200jk_incore_jk(h._h, _lib.dptr(dms), len(dms), nao, _lib.dptr(vj), _lib.dptr(vk)), 'b200jk_incore_jk')
        return (None if vj is None else vj.reshape(shape)), (None if vk is None else vk.reshape(shape))

    def close(self):
        self.handle.close()


def incore(mol, eri, dm, hermi=0, with_j=True, with_k=True, device=0, libpath=None):
    """_vhf.incore(eri, dm, hermi) (pyscf/scf/_vhf.py:283): one-shot J/K from stored integrals."""
    eng = IncoreJK(mol, eri, device=device, libpath=libpath)
    try:
        return eng.get_jk(dm, hermi, with_j, with_k)
    finally:
        eng.close()


def get_jk(mol, dm, hermi=1, vhfopt=None, with_j=True, with_k=True, omega=None):
    """Drop-in for pyscf.scf.hf.get_jk (pyscf/scf/hf.py:963): returns (vj, vk) shaped like dm."""
    if vhfopt is None:
        vhfopt = _opt_cache.get(mol, omega)
    return vhfopt.get_jk(dm, hermi, with_j, with_k)


def patch(mf, device=0, libpath=None):
    """Install the GPU builder as `mf.get_jk` on a PySCF SCF object (instance override).

    Keeps the reference semantics of SCF.get_jk (pyscf/scf/hf.py:2136-2160): one cached optimizer per omega (mf._opt there,
    mf._b200_opts here), dropped by mf.reset() (pyscf/scf/hf.py:2331: reset clears _opt) and rebuilt when the molecule's
    integral tables change."""
    cache = _OptCache()
    incore_eng = {}

    def _get_jk(mol=None, dm=None, hermi=1, with_j=True, with_k=True, omega=None):
        if mol is None:
            mol = mf.mol
        if dm is None:
            dm = mf.make_rdm1()
        # RHF.get_jk (pyscf/scf/hf.py:2499-2508): stored integrals (mf._eri) serve the plain Coulomb operator of the object's
        # own molecule; everything else goes to the direct path
        eri = getattr(mf, '_eri', None)
        if isinstance(eri, np.ndarray) and mol is mf.mol and effective_omega(mol, omega) == 0.0:
            eng = incore_eng.get('eng')
            if eng is None or incore_eng.get('eri') is not eri:
                if eng is not None:
                    eng.close()
                eng = incore_eng['eng'] = IncoreJK(mol, eri, device=device, libpath=libpath)
                incore_eng['eri'] = eri
            return eng.get_jk(dm, hermi, with_j, with_k)
        opt = cache.get(mol, omega, direct_scf_tol=getattr(mf, 'direct_scf_tol', 1e-13), device=device, libpath=libpath)
        return opt.get_jk(dm, hermi, with_j, with_k)

    _get_jk._b200_direct = True
    mf.get_jk = _get_jk
    mf._b200_opts = cache
    cls_reset = getattr(mf, 'reset', None)
    if cls_reset is not None and not getattr(cls_reset, '_b200_wrapped', False):
        def _reset(mol=None):
            cache.clear()
            if incore_eng.get('eng') is not None:
                incore_eng.pop('eng').close()
                incore_eng.pop('eri', None)
            return cls_reset(mol)
        _reset._b200_wrapped = True
        mf.reset = _reset
    return mf
