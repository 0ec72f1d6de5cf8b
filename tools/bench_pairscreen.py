"""Measure pair-screened DF J/K (DF(pair_tol=...)) against the dense tensor on one GPU.

Reports the card and its power limit, then for C60/def2-SVP, Taxol/def2-TZVP and (Gly)30/cc-pVDZ omega-B97X (the Coulomb tensor
plus its range_coulomb(0.3) child, get_jk + get_k(omega=0.3) per build) the kept column fraction, the tensor size, the setup
time, the wall-clock ms per build (median of `steps` after one warm-up), the device time of the DF-J and DF-K stages of the last
build (CUDA events) and the host bytes streamed per build, dense and at pair_tol = 1e-13 wherever the dense tensor fits.
Variants are alternated over the rounds, each rebuilt per round.

    python tools/bench_pairscreen.py [--rounds 2] [--steps 3] [--tol 1e-13] [--only c60,taxol,gly30] [--out FILE]
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


def _stages(d):
    st = d.stage_times()
    return {'dfj_ms': st['j_rho'][0] + st['j_acc'][0], 'dfk_ms': st['k_gemm1'][0] + st['k_slice'][0] + st['k_gemm2'][0]}


def one(geom, basis, tol, steps, omega=None):
    from pyscf_b200 import gto
    from pyscf_b200.df import DF
    from pyscf_b200.gto.mole import geometry
    mol = gto.M(atom=geometry(geom), basis=basis)
    dm = scf_like_density(mol.nao, mol.nelectron // 2)
    t0 = time.perf_counter()
    d = DF(mol, pair_tol=tol).build()
    tensors = [d] + ([d.range_coulomb(omega)] if omega else [])
    setup_s = time.perf_counter() - t0

    def build():
        d.get_jk(dm, hermi=1)
        if omega:
            d.get_jk(dm, hermi=1, with_j=False, omega=omega)

    build()
    t = []
    for _ in range(steps):
        t0 = time.perf_counter()
        build()
        t.append((time.perf_counter() - t0) * 1e3)
    rec = {'pair_tol': tol, 'setup_s': setup_s, 'ms_per_build': float(np.median(t)), 'tensors': []}
    for x in tensors:
        ncol, npair = x.pair_stats()
        naux = x.get_naoaux()
        rec['tensors'].append({'omega': x._effective_omega(), 'naux': naux, 'kept_fraction': ncol / npair,
                               'tensor_GB': naux * ncol * 8 / 1e9, 'row_split': x.row_split(), **_stages(x), **x.stream_stats()})
    d.reset()
    return rec


CONFIGS = {'c60': ('c60', 'def2-svp', None, (None, 'tol')),
           'taxol': ('taxol', 'def2-tzvp', None, (None, 'tol')),
           'gly30': ('gly30', 'cc-pvdz', 0.3, ('tol',))}     # dense: 197 + 81 GB, beyond one GPU and its host


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--rounds', type=int, default=2)
    ap.add_argument('--steps', type=int, default=3)
    ap.add_argument('--tol', type=float, default=1e-13)
    ap.add_argument('--only', default='c60,taxol,gly30')
    ap.add_argument('--out', default=None)
    a = ap.parse_args()
    rec = card()
    print(json.dumps(rec), flush=True)
    for name in a.only.split(','):
        geom, basis, omega, variants = CONFIGS[name]
        res = {str(v): [] for v in variants}
        for r in range(a.rounds if len(variants) > 1 else 1):
            for v in (variants if r % 2 == 0 else variants[::-1]):
                res[str(v)].append(one(geom, basis, a.tol if v == 'tol' else None, a.steps, omega))
                print(json.dumps({name: {str(v): res[str(v)][-1]}}), flush=True)
        rec[name] = res
    if a.out:
        with open(a.out, 'w') as f:
            json.dump(rec, f, indent=1)


if __name__ == '__main__':
    main()
