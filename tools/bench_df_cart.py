"""Measure DF J/K of C60/cc-pVDZ with spherical and with Cartesian AOs (mol.cart = True) on one GPU.

Reports the card and its power limit, then per convention nao, naux, the tensor size, the setup time (auxiliary basis, metric,
tensor), the wall-clock ms per DF.get_jk of the SCF-like orbital-tagged density (median of `steps` after one warm-up) and the
device time of the DF-J and DF-K stages of the last call (CUDA events).  The expectation: DF-J streams the tensor, so it scales
with naux * npair; DF-K with naux * nao^2 * nocc.  The two conventions are alternated over the rounds, each rebuilt per round.

    python tools/bench_df_cart.py [--rounds 2] [--steps 5] [--out FILE]
"""
import argparse
import json
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

from bench_outcore import card, scf_like_density  # noqa: E402


def one(cart, steps):
    from pyscf_b200 import gto
    from pyscf_b200.df import DF
    from pyscf_b200.gto.mole import geometry
    mol = gto.M(atom=geometry('c60'), basis='cc-pvdz', cart=cart)
    nao, nocc = mol.nao, mol.nelectron // 2
    dm = scf_like_density(nao, nocc)
    t0 = time.perf_counter()
    d = DF(mol, 'cc-pvdz-jkfit').build()
    naux = d.get_naoaux()
    setup_s = time.perf_counter() - t0
    d.get_jk(dm, hermi=1)
    t = []
    for _ in range(steps):
        t0 = time.perf_counter()
        d.get_jk(dm, hermi=1)
        t.append((time.perf_counter() - t0) * 1e3)
    st = d.stage_times()
    npair = nao * (nao + 1) // 2
    rec = {'cart': cart, 'nao': nao, 'naux': naux, 'nocc': nocc, 'tensor_GB': naux * npair * 8 / 1e9, 'setup_s': setup_s,
           'ms_per_get_jk': float(np.median(t)), 'dfj_ms': st['j_rho'][0] + st['j_acc'][0],
           'dfk_ms': st['k_gemm1'][0] + st['k_slice'][0] + st['k_gemm2'][0], 'row_split': d.row_split(),
           'naux_npair': float(naux) * npair, 'naux_nao2_nocc': float(naux) * nao * nao * nocc}
    d.reset()
    return rec


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--rounds', type=int, default=2)
    ap.add_argument('--steps', type=int, default=5)
    ap.add_argument('--out', default=None)
    a = ap.parse_args()
    rec = card()
    print(json.dumps(rec), flush=True)
    res = {'sph': [], 'cart': []}
    for r in range(a.rounds):
        for cart in ((False, True) if r % 2 == 0 else (True, False)):
            res['cart' if cart else 'sph'].append(one(cart, a.steps))
            print(json.dumps(res['cart' if cart else 'sph'][-1]), flush=True)
    s, c = res['sph'][-1], res['cart'][-1]
    rec.update(res)
    rec['ratio_cart_over_sph'] = {'dfj_ms': c['dfj_ms'] / s['dfj_ms'], 'naux_npair': c['naux_npair'] / s['naux_npair'],
                                  'dfk_ms': c['dfk_ms'] / s['dfk_ms'], 'naux_nao2_nocc': c['naux_nao2_nocc'] / s['naux_nao2_nocc']}
    print(json.dumps({'ratio_cart_over_sph': rec['ratio_cart_over_sph']}), flush=True)
    if a.out:
        with open(a.out, 'w') as f:
            json.dump(rec, f, indent=1)


if __name__ == '__main__':
    main()
