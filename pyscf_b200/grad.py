"""Nuclear-gradient J/K on H100: the role of pyscf.grad.rhf.get_jk / get_j / get_k (pyscf/grad/rhf.py:191-235)

    vj[x, i, j] = - sum_kl (nabla_x i  j | k l) D_lk            vk[x, i, l] = - sum_jk (nabla_x i  j | k l) D_jk

(libcint `int2e_ip1`, 3 components, the derivative acting on the electron coordinate of the first function), which the
reference contracts with `_vhf.direct_mapdm(intor='int2e_ip1', 's2kl', ('lk->s1ij', 'jk->s1il'), ...)`.

No derivative-integral kernels are needed.  For a contracted Cartesian Gaussian b_a = x^ax y^ay z^az sum_k c_k exp(-alpha_k r^2)

    d/dx b_a = ax * b_(a - 1x)[c]  -  b_(a + 1x)[2 alpha c]

so (nabla_x i j|kl) is a combination of ORDINARY integrals over two companion shells of i's shell: one unit of angular momentum
up with the coefficients 2 alpha_k c_k, one down with c_k.  The J/K kernels of the 4-center path work on bare Cartesian
monomials anyway, hence: build the molecule extended by the companion shells as Cartesian AOs (mol.cart, b200jk_create2), embed the
density in the original block, run ONE ordinary J/K build there, and read the gradient matrices off the (companion, original)
blocks: vj[x][i,j] = -(T (ax J[a-,b] - J[a+,b]) T^T)_ij with the cart->sph matrices T of the two shells.  The quartets whose
density blocks vanish (companion x companion) are dropped by the on-device screening.
Limits: the companion of an f shell is a g shell, beyond the 4-center kernel classes: original shells up to d (cc-pVDZ, def2-SVP, 6-31G*).
"""
import math

import numpy as np

from .jk import VHFOpt

ANG_OF, NPRIM_OF, NCTR_OF, PTR_EXP, PTR_COEFF = 1, 2, 3, 5, 6
_FAC = {0: 0.282094791773878143, 1: 0.488602511902919921}


def _fac(l):
    """angular factor libcint folds into its s and p functions (pyscf/gto/mole.py:159-181)"""
    return _FAC.get(l, 1.0)


def cart_comps(l):
    """libcint Cartesian order: lx descending, then ly descending (pyscf/lib/parameters.py:69-77)"""
    return [(x, y, l - x - y) for x in range(l, -1, -1) for y in range(l - x, -1, -1)]


def cart2sph(l):
    """T[m, a]: real solid harmonics (libcint order: p = x,y,z; l >= 2: m = -l..l) in bare Cartesian monomials, orthonormal on the
    sphere (Helgaker, Jorgensen, Olsen, eq. 6.4.47) — the matrices the library uses for its density / J,K transforms."""
    comps = cart_comps(l)
    nc = len(comps)
    if l == 0:
        return np.array([[_FAC[0]]])
    if l == 1:
        return np.eye(3) * _FAC[1]
    T = np.zeros((2 * l + 1, nc))
    ang = math.sqrt((2 * l + 1) / (4.0 * math.pi))
    f = math.factorial

    def binom(n, k):
        return 0.0 if k < 0 or k > n else float(math.comb(n, k))

    for m in range(-l, l + 1):
        am = abs(m)
        N = 1.0 / (2.0 ** am * f(l)) * math.sqrt(2.0 * f(l + am) * f(l - am) / (2.0 if m == 0 else 1.0))
        two_vm = 1 if m < 0 else 0
        for t in range((l - am) // 2 + 1):
            for u in range(t + 1):
                vmax2 = 2 * int(math.floor(am / 2.0 - two_vm / 2.0)) + two_vm
                for two_v in range(two_vm, vmax2 + 1, 2):
                    sp = t + (two_v - two_vm) // 2
                    cf = (-1.0) ** sp * 0.25 ** t * binom(l, t) * binom(l - t, am + t) * binom(t, u) * binom(am, two_v)
                    lx, ly, lz = 2 * t + am - 2 * u - two_v, 2 * u + two_v, l - 2 * t - am
                    if lx < 0 or ly < 0 or lz < 0:
                        continue
                    T[m + l, comps.index((lx, ly, lz))] += ang * N * cf
    return T


class _Ext:
    """The molecule extended by the derivative companions of every shell, as Cartesian AOs: shells [originals | l+1 | l-1]."""

    def __init__(self, mol):
        if getattr(mol, 'cart', False):
            raise NotImplementedError('gradient J/K of a cart=True molecule')
        bas = np.asarray(mol._bas, dtype=np.int32)
        env = list(np.asarray(mol._env, dtype=np.float64))
        if int(bas[:, ANG_OF].max()) > 2:
            raise NotImplementedError('gradient J/K needs the (l+1) companion of every shell: orbital shells up to d only '
                                      '(an f shell would need (g.|..) kernel classes)')
        plus, minus = [], []
        for b in bas:
            l, npr, nct = int(b[ANG_OF]), int(b[NPRIM_OF]), int(b[NCTR_OF])
            ex = np.array(env[b[PTR_EXP]:b[PTR_EXP] + npr])
            cf = np.array(env[b[PTR_COEFF]:b[PTR_COEFF] + npr * nct]).reshape(nct, npr)
            for dl, coef in ((1, 2.0 * ex * cf), (-1, cf)):
                if l + dl < 0:
                    continue
                nb = b.copy()
                nb[ANG_OF] = l + dl
                nb[PTR_COEFF] = len(env)
                env.extend((coef / _fac(l + dl)).ravel())      # the library multiplies s, p functions by fac: keep bare monomials
                (plus if dl > 0 else minus).append(nb)
        self.nbas0 = len(bas)
        self.plus_of = {i: self.nbas0 + k for k, i in enumerate(range(self.nbas0))}
        has_minus = [i for i in range(self.nbas0) if bas[i, ANG_OF] > 0]
        self.minus_of = {i: self.nbas0 + len(plus) + k for k, i in enumerate(has_minus)}
        ext = mol.copy()
        ext._bas = np.ascontiguousarray(np.vstack([bas] + [np.array(plus)] + ([np.array(minus)] if minus else [])), dtype=np.int32)
        ext._env = np.array(env, dtype=np.float64)
        ext.nbas = len(ext._bas)
        ext.cart = True
        self.mol = ext
        self.loc = ext.ao_loc_nr(cart=True)             # Cartesian AO offsets of the extended shells
        self.n0 = int(self.loc[self.nbas0])               # Cartesian functions of the original shells
        self.loc_sph = mol.ao_loc_nr(cart=False)
        self.bas = bas
        # spherical <- bare Cartesian of the original block, and the fac scaling of the library's Cartesian functions
        nao = int(self.loc_sph[-1])
        self.T = np.zeros((nao, self.n0))
        for i, b in enumerate(bas):
            l, nct = int(b[ANG_OF]), int(b[NCTR_OF])
            t = cart2sph(l)
            ns, nc = t.shape
            for c in range(nct):
                self.T[self.loc_sph[i] + c * ns:self.loc_sph[i] + (c + 1) * ns, self.loc[i] + c * nc:self.loc[i] + (c + 1) * nc] = t
        # library function = fac * bare function: fac(l) on the original shells (libcint's s, p factors), 1 on the companions
        # (their coefficients were divided by fac above)
        self.fac = np.ones(int(self.loc[-1]))
        for i in range(self.nbas0):
            self.fac[self.loc[i]:self.loc[i + 1]] = _fac(int(bas[i, ANG_OF]))


def _assemble(ext, M):
    """Gradient matrices from a J- or K-like matrix M[p, q] = (b_p . | . b_q) over bare Cartesian functions of the extended basis
    (rows: companions, columns: original block): out[x, i, j] = -(nabla_x i . | . j), spherical i, j."""
    nao = ext.T.shape[0]
    G = np.zeros((3, ext.n0, ext.n0))
    for i, b in enumerate(ext.bas):
        l, nct = int(b[ANG_OF]), int(b[NCTR_OF])
        comps = cart_comps(l)
        up = {c: k for k, c in enumerate(cart_comps(l + 1))}
        dn = {c: k for k, c in enumerate(cart_comps(l - 1))} if l > 0 else {}
        nc, ncu, ncd = len(comps), len(up), len(dn)
        pu, pd = ext.loc[ext.plus_of[i]], (ext.loc[ext.minus_of[i]] if l > 0 else 0)
        for c in range(nct):
            for a, pw in enumerate(comps):
                row = ext.loc[i] + c * nc + a
                for x in range(3):
                    hi = list(pw)
                    hi[x] += 1
                    g = -M[pu + c * ncu + up[tuple(hi)], :ext.n0]
                    if pw[x] > 0:
                        lo = list(pw)
                        lo[x] -= 1
                        g = g + pw[x] * M[pd + c * ncd + dn[tuple(lo)], :ext.n0]
                    G[x, row] = g
    return -np.einsum('ia,xab,jb->xij', ext.T, G, ext.T).reshape(3, nao, nao)


def get_jk(mol, dm, with_j=True, with_k=True, device=0, libpath=None, direct_scf_tol=1e-13):
    """(vj, vk), each [3, nao, nao] (or [n_dm, 3, nao, nao] for a stack of densities), pyscf/grad/rhf.py:191-205.  dm must be
    symmetric (the reference's 's2kl' contraction and 'lk->s1ij' script assume it as well)."""
    dm = np.asarray(dm, dtype=np.float64)
    nao = int(mol.ao_loc_nr(cart=False)[-1])
    shape = dm.shape
    dms = dm.reshape(-1, nao, nao)
    if abs(dms - dms.transpose(0, 2, 1)).max() > 1e-10 * max(1.0, abs(dms).max()):
        raise RuntimeError('grad.get_jk: the density matrix must be symmetric')
    ext = _Ext(mol)
    n = int(ext.loc[-1])
    dext = np.zeros((len(dms), n, n))
    f0 = ext.fac[:ext.n0]
    for s, d in enumerate(dms):
        dext[s, :ext.n0, :ext.n0] = ext.T.T.dot(d).dot(ext.T) / np.outer(f0, f0)
    opt = VHFOpt(ext.mol, direct_scf_tol=direct_scf_tol, device=device, libpath=libpath)
    try:
        vj, vk = opt.get_jk(dext, hermi=1, with_j=with_j, with_k=with_k)
    finally:
        opt.close()
    scale = np.outer(ext.fac, ext.fac)
    outj = np.array([_assemble(ext, m / scale) for m in vj]) if with_j else None
    outk = np.array([_assemble(ext, m / scale) for m in vk]) if with_k else None
    if len(shape) == 2:
        outj = None if outj is None else outj[0]
        outk = None if outk is None else outk[0]
    return outj, outk


def get_j(mol, dm, **kw):
    """pyscf/grad/rhf.py:207-220"""
    return get_jk(mol, dm, with_k=False, **kw)[0]


def get_k(mol, dm, **kw):
    """pyscf/grad/rhf.py:222-235"""
    return get_jk(mol, dm, with_j=False, **kw)[1]


def get_veff(mol, dm, **kw):
    """pyscf/grad/rhf.py:237-240: vj - vk/2"""
    vj, vk = get_jk(mol, dm, **kw)
    return vj - vk * 0.5
