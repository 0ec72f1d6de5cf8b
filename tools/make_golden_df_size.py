#!/usr/bin/env python
"""Oracle parity fixtures of the density-fitting path AT CONFIGURATION SIZE (BASELINE.json configs 3-5): C60/def2-SVP,
Taxol/def2-TZVP, (Gly)30/cc-pVDZ (Coulomb tensor and the erf(0.3 r)/r tensor of omega-B97X).  Run in the build container
(CPU oracle, pinned by tests/test_oracle_golden.py); the .npz files are committed under tests/golden/.

The full tensors (12.7 / 111 / 197 GB) are beyond the oracle, but cderi = L^-1 (P|mu nu) is separable in the AO-pair
column, and J/K of a density SUPPORTED ON A FEW SHELLS S only need the slab (P|s nu), s in S:
  * `cols` / `cderi_cols`: a sample of AO-pair columns (two shell pairs of every angular-momentum pair type, a few
    components each) of the oracle tensor, all naux rows: checks the 3-center kernels of every class, the metric, its
    factorisation and the triangular solve, the row sharding and the tensor layout.
  * slab density  C_S[nao, nocc] (non-zero rows only on the AOs of S, nocc = the configuration's nocc, so that the
    contraction lengths of both GEMM stages are the real ones), D_S = C_S C_S^T:
        K[i,l]  = sum_P sum_{j,k in S} B[P,i,j] D_S[j,k] B[P,k,l]     every element of K, from the slab alone
        J[s,nu] = sum_P B[P,s,nu] rho_P,  rho_P = sum_{j,k in S} B[P,j,k] D_S[j,k]    the rows s in S of J
    stored as `vk_idx`/`vk_val` (sampled elements), fp(K), and the J rows.  Both K engines (int8 slices on the
    orbital tag, FP64 general path on the bare matrix) are compared with these on the GPU (tests/test_df_size.py, bench.py).
Cartesian cases (name in CART, mol.cart = True) take their integrals from tests/cart_oracle.py, the oracle library's Cartesian
entry points, and also report the metric's condition number and the spread of the slab J/K when the 3-center and metric
integrals carry 1e-15 relative noise: how well the Cartesian problem itself defines J/K (Cartesian auxiliary bases are much
worse conditioned than spherical ones), which sets the bar of the GPU comparison.
Usage: python tools/make_golden_df_size.py [c60 taxol taxol_svp gly30 gly30_lr c60_cart]
"""
import os
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import numpy as np            # noqa: E402
import scipy.linalg           # noqa: E402
from pyscf_b200 import gto    # noqa: E402
from pyscf_b200.gto.mole import geometry, make_auxmol   # noqa: E402
from oracle import oracle as O   # noqa: E402

CASES = {   # name: (geometry, basis, nocc, omega)
    'c60': ('c60', 'def2-svp', 180, None),
    'taxol': ('taxol', 'def2-tzvp', 226, None),
    # one GPU of 80 GB holds its 28 GB tensor but not the int8 slices of all its rows: resident and re-cut slices both run
    'taxol_svp': ('taxol', 'def2-svp', 226, None),
    'gly30': ('gly30', 'cc-pvdz', 455, None),
    'gly30_lr': ('gly30', 'cc-pvdz', 455, 0.3),
    'gly4': ('gly4', 'cc-pvdz', 65, None),          # small: the same fixture at a size the CPU tests can build in full
    'c60_cart': ('c60', 'cc-pvdz', 180, None),      # Cartesian AOs and auxiliary functions: nao 900, naux 4860
}
CART = {'c60_cart'}
NOISE = 1e-15         # relative noise of the integrals in the conditioning probe of the Cartesian cases
# fixtures kept below 1 MB: one shell pair per angular-momentum pair type, two components each, fewer sampled K elements
SMALL = {'taxol_svp', 'c60_cart'}


def slab_coeff(nao, nocc, sao, seed=7):
    """C_S: random normal on the rows `sao`, zero elsewhere (the tests rebuild it from the stored seed)."""
    rng = np.random.RandomState(seed)
    c = np.zeros((nao, nocc))
    c[sao] = rng.standard_normal((len(sao), nocc)) / np.sqrt(nocc)
    return c


def pick_pairs(mol, rng, per_type=2):
    """Two shell pairs (ish >= jsh) of every (l_i, l_j) type, spread over the molecule; the two shells sit on the same atom
    or on atoms closer than 2.2 Angstrom (a pair of distant shells has a vanishing tensor column, which checks nothing)."""
    ls, at = mol._bas[:, 1], mol._bas[:, 0]
    coords = np.array([mol._env[mol._atm[a, 1]:mol._atm[a, 1] + 3] for a in range(mol.natm)])
    out = []
    for la in sorted(set(ls)):
        for lb in sorted(set(ls)):
            if lb > la:
                continue
            ia, ib_all = np.where(ls == la)[0], np.where(ls == lb)[0]
            got = set()
            for _ in range(200):
                i = int(rng.choice(ia))
                near = ib_all[np.linalg.norm(coords[at[ib_all]] - coords[at[i]], axis=1) < 2.2 / 0.52917721092]
                ib = near if len(near) else ib_all
                j = int(rng.choice(ib))
                if i < j:
                    i, j = j, i
                if (i, j) not in got:
                    got.add((i, j))
                if len(got) >= per_type:
                    break
            out += sorted(got)
    return out


def pick_slab_shells(mol, rng):
    """One shell of every angular momentum on two different atoms (the second set far from the first)."""
    ls, at = mol._bas[:, 1], mol._bas[:, 0]
    coords = np.array([mol._env[mol._atm[a, 1]:mol._atm[a, 1] + 3] for a in range(mol.natm)])
    a0 = int(rng.randint(mol.natm))
    a1 = int(np.argmax(np.linalg.norm(coords - coords[a0], axis=1)))
    shells = []
    for l in sorted(set(ls)):
        for a in (a0, a1):
            cand = np.where((ls == l) & (at == a))[0]
            if len(cand) == 0:      # e.g. no f shell on a hydrogen: take the nearest atom that has one
                cand_all = np.where(ls == l)[0]
                d = np.linalg.norm(coords[at[cand_all]] - coords[a], axis=1)
                cand = cand_all[[int(np.argmin(d))]]
            shells.append(int(cand[len(cand) // 2]))
    return sorted(set(shells))


def slab_jk(B, S, c0, mol, loc, sao, d_ss):
    """J rows of the slab AOs and all of K for the density D_SS on the slab AOs, from the slab tensor B[P, (s, nu) blocks]."""
    naux, nao = B.shape[0], int(loc[-1])
    Bs = np.empty((naux, len(sao), nao))                       # reorder to B[P, s_ao, nu]
    row = 0
    for si, s in enumerate(S):
        ds = loc[s + 1] - loc[s]
        for j in range(mol.nbas):
            p = si * mol.nbas + j
            dj = loc[j + 1] - loc[j]
            Bs[:, row:row + ds, loc[j]:loc[j + 1]] = B[:, c0[p]:c0[p] + ds * dj].reshape(naux, ds, dj)
        row += ds
    rho = np.einsum('psk,sk->p', Bs[:, :, sao], d_ss)
    vj_rows = np.einsum('p,psn->sn', rho, Bs)                  # J[s, :] for s in sao
    vk = np.zeros((nao, nao))
    blk = 256
    for p0 in range(0, naux, blk):
        b = Bs[p0:p0 + blk]                                    # [pb, ns, nao]
        t = np.matmul(d_ss, b)                                 # D_SS B_P[S,:]   [pb, ns, nao]
        vk += b.reshape(-1, nao).T.dot(t.reshape(-1, nao))     # sum_{P,s} B[P,s,i] T[P,s,n]  (BLAS)
    return vj_rows, vk


def main(name):
    geom, basis, nocc, omega = CASES[name]
    cart = name in CART
    mol = gto.M(atom=geometry(geom), basis=basis, cart=cart)
    auxmol = make_auxmol(mol)
    if cart:
        sys.path.insert(0, os.path.join(ROOT, 'tests'))
        import cart_oracle as C
        int2c2e, int3c2e_pairs = C.int2c2e, C.int3c2e_pairs
    else:
        int2c2e, int3c2e_pairs = O.int2c2e, O.int3c2e_pairs
    nao, naux = mol.nao, auxmol.nao
    loc = mol.ao_loc_nr()
    rng = np.random.RandomState(11)
    t0 = time.time()
    if omega is not None:
        mol._env[8] = omega
    j2c = int2c2e(auxmol, omega=mol._env[8])
    cond = 0.0
    try:
        low = scipy.linalg.cholesky(j2c, lower=True)
        chol = 1
        print(name, 'nao', nao, 'naux', naux, 'j2c + cholesky %.1f s' % (time.time() - t0), 'cond estimate %.2e'
              % (np.abs(np.diag(low)).max() / np.abs(np.diag(low)).min()) ** 2, flush=True)
        if cart:
            w = scipy.linalg.eigvalsh(j2c)
            cond = float(w[-1] / w[0])
            print('  metric condition number %.3e (eigenvalues %.3e .. %.3e)' % (cond, w[0], w[-1]), flush=True)

        def solve(x):
            return scipy.linalg.solve_triangular(low, x, lower=True, overwrite_b=True)
    except scipy.linalg.LinAlgError:
        # the reference's fallback (pyscf/df/incore.py:150-158, _eig_decompose :263-270): cderi = diag(w)^-1/2 V^T (P|mu nu), w > lindep.
        # The rows are then only defined up to rotations inside near-degenerate eigenspaces: compare J/K, not the tensor.
        w, v = scipy.linalg.eigh(j2c)
        mask = w > 1e-7
        winv = (v[:, mask] / np.sqrt(w[mask])).T
        chol = 0
        print(name, 'nao', nao, 'naux', naux, 'metric not positive definite: eigen-decomposition, %d of %d kept (w > 1e-7), smallest kept %.3e, '
              'largest dropped %.3e, %.1f s' % (mask.sum(), naux, w[mask].min(), w[~mask].max() if (~mask).any() else 0.0, time.time() - t0), flush=True)
        naux = int(mask.sum())

        def solve(x):
            return winv.dot(x)
    # ---- sampled columns
    small = name in SMALL
    pairs = pick_pairs(mol, rng, per_type=1 if small else 2)
    t0 = time.time()
    j3c, col0 = int3c2e_pairs(mol, auxmol, pairs)
    cd = solve(j3c.copy())
    cols, keep = [], []
    for p, (i, j) in enumerate(pairs):
        di, dj = loc[i + 1] - loc[i], loc[j + 1] - loc[j]
        comps = [(a, b) for a in range(di) for b in range(dj) if loc[i] + a >= loc[j] + b]
        for idx in rng.choice(len(comps), size=min(2 if small else 3, len(comps)), replace=False):
            a, b = comps[idx]
            mu, nu = loc[i] + a, loc[j] + b
            cols.append(mu * (mu + 1) // 2 + nu)
            keep.append(col0[p] + a * dj + b)
    cols, keep = np.array(cols), np.array(keep)
    cderi_cols = np.ascontiguousarray(cd[:, keep])
    print('  %d shell pairs, %d sampled columns, %.1f s' % (len(pairs), len(cols), time.time() - t0), flush=True)
    # ---- slab density
    S = pick_slab_shells(mol, rng)
    sao = np.concatenate([np.arange(loc[s], loc[s + 1]) for s in S])
    t0 = time.time()
    slab_pairs = [(s, j) for s in S for j in range(mol.nbas)]
    j3s, c0 = int3c2e_pairs(mol, auxmol, slab_pairs)
    B = solve(j3s.copy())     # [naux, sum_s d_s * nao]
    print('  slab: shells', S, '->', len(sao), 'AOs, %.1f s' % (time.time() - t0), flush=True)
    t0 = time.time()
    c_s = slab_coeff(nao, nocc, sao)
    d_ss = 2.0 * c_s[sao].dot(c_s[sao].T)                      # occupation 2, as bench.py's SCF-like density
    vj_rows, vk = slab_jk(B, S, c0, mol, loc, sao, d_ss)
    print('  J rows / K from the slab %.1f s; |K|max %.3g |J|max %.3g' % (time.time() - t0, abs(vk).max(), abs(vj_rows).max()), flush=True)
    extra = {}
    if cart:
        # conditioning probe: the same J/K from integrals with NOISE relative noise (three draws), against the clean result
        spread_j = spread_k = spread_c = 0.0
        for seed in range(3):
            nz = np.random.RandomState(100 + seed)
            j2n = j2c * (1 + NOISE * nz.standard_normal(j2c.shape))
            j2n = 0.5 * (j2n + j2n.T)
            lown = scipy.linalg.cholesky(j2n, lower=True)
            cdn = scipy.linalg.solve_triangular(lown, j3c * (1 + NOISE * nz.standard_normal(j3c.shape)), lower=True)[:, keep]
            spread_c = max(spread_c, float(abs(cdn - cderi_cols).max()))
            Bn = scipy.linalg.solve_triangular(lown, j3s * (1 + NOISE * nz.standard_normal(j3s.shape)), lower=True)
            vjn, vkn = slab_jk(Bn, S, c0, mol, loc, sao, d_ss)
            spread_j = max(spread_j, float(abs(vjn - vj_rows).max()))
            spread_k = max(spread_k, float(abs(vkn - vk).max()))
            print('  noise probe %d: max |dJ| %.2e  max |dK| %.2e  max |d cderi_cols| %.2e (running maxima)'
                  % (seed, spread_j, spread_k, spread_c), flush=True)
        extra = dict(cond=cond, noise=NOISE, noise_dj=spread_j, noise_dk=spread_k, noise_dcol=spread_c)
    del j3s, B
    nsamp = 3000 if small else 6000
    ii, ll = rng.randint(nao, size=nsamp), rng.randint(nao, size=nsamp)
    ii[:len(sao)] = sao
    ll[:len(sao)] = sao[::-1]
    out = os.path.join(ROOT, 'tests', 'golden', 'df_size_%s.npz' % name)
    np.savez_compressed(out, nao=nao, naux=naux, nocc=nocc, omega=0.0 if omega is None else omega,
                        cols=cols, cderi_cols=cderi_cols, chol=chol, slab_shells=np.array(S), sao=sao, seed=7,
                        vj_rows=vj_rows, vk_idx=np.stack([ii, ll], 1), vk_val=vk[ii, ll], vk_fp=O.fp(vk), vk_absmax=abs(vk).max(),
                        vk_diag=np.diag(vk).copy(), **extra)
    print('  wrote', out, '%.1f MB' % (os.path.getsize(out) / 1e6), flush=True)


if __name__ == '__main__':
    for n in (sys.argv[1:] or ['c60', 'taxol', 'gly30', 'gly30_lr']):
        main(n)
