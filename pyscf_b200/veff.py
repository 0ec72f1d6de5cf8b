"""`get_veff` on top of the GPU J/K builders: the callers one level above `get_jk` on the hot path.

Mirrors (argument meaning, incremental-Fock behaviour, the `ecoul` / `vj` / `vk` tags the SCF loop reads back):
  * scf.hf.SCF.get_veff      pyscf/scf/hf.py:2172-2201   vhf = J - K/2, built from D - D_last when direct_scf
  * scf.uhf.UHF.get_veff     pyscf/scf/uhf.py:1066-1095  vhf[s] = J[a] + J[b] - K[s]
  * dft.rks.get_veff         pyscf/dft/rks.py:37-142     J/K part only: hybrid and range-separated mixes
                                                         K = hyb K + (alpha - hyb) K_LR(omega)   (:105-127)
The exchange-correlation quadrature (numint / libxc) is outside the hot path (SURVEY.md §8): `get_veff_rks` takes the
functional's (omega, alpha, hyb) and an optional callable returning (n, exc, vxc) and adds the J/K terms to it.

`get_jk` everywhere is a callable with the reference's signature
`get_jk(mol, dm, hermi=1, with_j=True, with_k=True, omega=None) -> (vj, vk)` — e.g. the closure installed by
`pyscf_b200.jk.patch`, `functools.partial(pyscf_b200.jk.get_jk, ...)` or `make_get_jk(mol)` below.
"""
import numpy as np

# (omega, alpha, hyb) as returned by ni.rsh_and_hybrid_coeff (pyscf/dft/numint.py; values are libxc's, which is not
# part of the reference tree): alpha = long-range HF fraction, hyb = short-range HF fraction.
RSH_AND_HYBRID_COEFF = {
    'hf': (0.0, 0.0, 1.0),
    'lda': (0.0, 0.0, 0.0), 'pbe': (0.0, 0.0, 0.0), 'blyp': (0.0, 0.0, 0.0),
    'b3lyp': (0.0, 0.0, 0.2), 'pbe0': (0.0, 0.0, 0.25),
    'hse06': (0.11, 0.0, 0.25),
    'camb3lyp': (0.33, 0.65, 0.19),
    'wb97x': (0.3, 1.0, 0.157706),
    'wb97xd': (0.2, 1.0, 0.222036),
    'lcwpbe': (0.4, 1.0, 0.0),
}


class TaggedArray(np.ndarray):
    """ndarray with attributes, the role of lib.tag_array (pyscf/lib/numpy_helper.py) for vhf.ecoul / .vj / .vk."""

    def __new__(cls, a, **tags):
        obj = np.asarray(a).view(cls)
        obj.__dict__.update(tags)
        return obj

    # tags (ecoul, vj, vk) describe this array only: results of arithmetic come back untagged, as lib.tag_array's
    # NPArrayWithTag.__array_wrap__ does (pyscf/lib/numpy_helper.py:1477-1484)
    def __array_wrap__(self, out, context=None, return_scalar=False):
        if out.ndim == 0:
            return out[()]
        return out.view(np.ndarray)


def tag_array(a, **tags):
    return TaggedArray(a, **tags)


def make_get_jk(mol, device=0, direct_scf_tol=1e-13, libpath=None, with_df=None):
    """A get_jk callable with one cached optimizer per omega (SCF._opt, pyscf/scf/hf.py:1803,2141-2146); routes to
    `with_df.get_jk` when a DF object is given (_DFHF.get_jk, pyscf/df/df_jk.py:150-179)."""
    from .jk import VHFOpt
    opts = {}

    def get_jk(mol_=None, dm=None, hermi=1, with_j=True, with_k=True, omega=None):
        if with_df is not None:
            return with_df.get_jk(dm, hermi, with_j, with_k, direct_scf_tol, omega)
        key = omega or None
        if key not in opts:
            opts[key] = VHFOpt(mol, direct_scf_tol=direct_scf_tol, omega=omega, device=device, libpath=libpath)
        return opts[key].get_jk(dm, hermi, with_j, with_k)

    get_jk.opts = opts
    return get_jk


def get_veff_rhf(get_jk, mol, dm, dm_last=None, vhf_last=None, hermi=1, direct_scf=True):
    """RHF effective potential J - K/2 (pyscf/scf/hf.py:2172-2201).  With direct_scf and a previous (dm_last, vhf_last)
    only the density CHANGE is contracted — the Schwarz x density screening then discards most quartets late in the SCF."""
    dm = np.asarray(dm)
    if not direct_scf or dm_last is None:
        vj, vk = get_jk(mol, dm, hermi)
        vhf = vj - vk * .5
        if dm.ndim == 2:
            vhf = tag_array(vhf, ecoul=np.einsum('ij,ji->', dm, vj).real * .5)
        return vhf
    assert vhf_last is not None
    dm_last = np.asarray(dm_last)
    ddm = dm - dm_last
    vj, vk = get_jk(mol, ddm, hermi)
    vhf = vj - vk * .5
    vhf = vhf + np.asarray(vhf_last)
    if hasattr(vhf_last, 'ecoul') and dm.ndim == 2:
        # Ecoul = Ecoul_last + dm_last.J[ddm] + 1/2 ddm.J[ddm]                        (hf.py:2189-2196)
        ecoul = np.einsum('ij,ji->', dm_last, vj).real + np.einsum('ij,ji->', ddm, vj).real * .5 + vhf_last.ecoul
        vhf = tag_array(vhf, ecoul=ecoul)
    return vhf


def get_veff_uhf(get_jk, mol, dm, dm_last=None, vhf_last=None, hermi=1, direct_scf=True):
    """UHF effective potential vhf[s] = J[alpha] + J[beta] - K[s] (pyscf/scf/uhf.py:1066-1095); dm = (dm_alpha, dm_beta)."""
    dm = np.asarray(dm)
    if dm.ndim == 2:      # "Treat dm as RHF density matrix" (uhf.py:1069-1071)
        dm = np.repeat(dm[None] * .5, 2, axis=0)
    incremental = direct_scf and dm_last is not None
    ddm = dm - np.asarray(dm_last) if incremental else dm
    vj, vk = get_jk(mol, ddm, hermi)
    vj = vj[0] + vj[1]
    vhf = vj - vk
    if not incremental:
        if dm.ndim == 3:      # a single (alpha, beta) pair; batches of pairs carry no energy tag (uhf.py:1076-1078)
            vhf = tag_array(vhf, ecoul=np.einsum('nij,ji->', dm, vj).real * .5)
        return vhf
    assert vhf_last is not None
    vhf = vhf + np.asarray(vhf_last)
    if hasattr(vhf_last, 'ecoul') and dm.ndim == 3:
        ecoul = (np.einsum('nij,ji->', np.asarray(dm_last), vj).real + np.einsum('nij,ji->', ddm, vj).real * .5
                 + vhf_last.ecoul)
        vhf = tag_array(vhf, ecoul=ecoul)
    return vhf


def get_vjk_rks(get_jk, mol, dm, omega=0.0, alpha=0.0, hyb=0.0, hermi=1):
    """The J and exchange matrices an RKS Fock build needs for a functional with coefficients (omega, alpha, hyb)
    (pyscf/dft/rks.py:98-127).  Returns (vj, vk) with vk already mixed, vk None for pure functionals."""
    if abs(hyb) < 1e-10 and abs(alpha) < 1e-10:
        return get_jk(mol, dm, hermi, with_k=False)[0], None
    if omega == 0:
        vj, vk = get_jk(mol, dm, hermi)
        vk = vk * hyb
    elif alpha == 0:      # LR = 0: short-range exchange only (HSE-type)
        vj = get_jk(mol, dm, hermi, with_k=False)[0]
        vk = get_jk(mol, dm, hermi, with_j=False, omega=-omega)[1] * hyb
    elif hyb == 0:        # SR = 0: long-range exchange only (LC-type)
        vj = get_jk(mol, dm, hermi, with_k=False)[0]
        vk = get_jk(mol, dm, hermi, with_j=False, omega=omega)[1] * alpha
    else:                 # SR and LR exchange with different ratios (wB97X, CAM-B3LYP)
        vj, vk = get_jk(mol, dm, hermi)
        vk = vk * hyb
        vk = vk + get_jk(mol, dm, hermi, with_j=False, omega=omega)[1] * (alpha - hyb)
    return vj, vk


def get_veff_rks(get_jk, mol, dm, xc='b3lyp', dm_last=None, vhf_last=None, hermi=1, direct_scf=True, nr_rks=None):
    """RKS effective potential Vxc + J - K/2 (pyscf/dft/rks.py:37-142) with the J/K part on the GPU.

    nr_rks(dm) -> (nelec, exc, vxc) supplies the quadrature of the semilocal part (the reference's ni.nr_rks, :82); when
    None the semilocal term is zero, which leaves exactly the Coulomb + exact-exchange potential the benchmark times.
    `xc` is a key of RSH_AND_HYBRID_COEFF or an (omega, alpha, hyb) tuple.  The result carries ecoul, exc, vj, vk like the
    reference's (:134-141) so the next call can be incremental (:98-103)."""
    omega, alpha, hyb = RSH_AND_HYBRID_COEFF[xc.lower().replace('-', '')] if isinstance(xc, str) else xc
    dm = np.asarray(dm)
    ground_state = dm.ndim == 2
    if hermi == 2 or nr_rks is None:
        n, exc, vxc = 0, 0.0, np.zeros_like(dm)
    else:
        n, exc, vxc = nr_rks(dm)
        vxc = np.array(vxc, dtype=np.float64, copy=True)
    incremental = direct_scf and dm_last is not None and getattr(vhf_last, 'vj', None) is not None
    _dm = dm - np.asarray(dm_last) if incremental else dm
    vj, vk = get_vjk_rks(get_jk, mol, _dm, omega, alpha, hyb, hermi)
    if incremental:
        vj = vj + vhf_last.vj
        if vk is not None:
            vk = vk + vhf_last.vk
    if vk is None:
        vxc = vxc + vj
    else:
        vxc = vxc + vj - vk * .5
        if ground_state:
            exc -= np.einsum('ij,ji', dm, vk).real * .5 * .5
    ecoul = np.einsum('ij,ji', dm, vj).real * .5 if ground_state else None
    return tag_array(vxc, ecoul=ecoul, exc=exc, vj=vj, vk=vk)
