"""Measure direct RPA on one GPU (pyscf_b200.rpa: b200jk_df_rpa, df_rpa.cuh).

Workloads (random orthonormal orbitals and synthetic energies, occupied < 0 < virtual: the time does not depend on the values),
all at nw = 40:
  bz_tz_rpa    benzene/cc-pVTZ, RPA
  c60_rpa      C60/def2-SVP, RPA (nocc 180, nvir 660, naux 4500)
  c60_urpa     C60/def2-SVP, URPA with nocc_beta = nocc_alpha - 1
Per workload: the card name and power limit (read in the same process), the device time of stage 1, of the Pi GEMMs and of the
factorisations (CUDA events inside the library, summed over the frequencies), the FLOPs of stage 1 and of the executed
upper-triangle Pi tiles counted here from the shapes, the achieved FP64 TFLOP/s, and the end-to-end wall time of the call
(median of `--steps` after one warm-up call).
Yardstick in the same process: torch fp64 (L chi) @ L^T plus torch.linalg.cholesky of I - Pi for one frequency on the same
shapes (cuBLAS / cuSOLVER), scaled by nw.

    python tools/bench_df_rpa.py [--steps 3] [--only bz_tz_rpa,c60_rpa,c60_urpa] [--out FILE]
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

from bench_outcore import card  # noqa: E402

NW = 40
BM = 64     # CTA tile of the Pi GEMM (df_ao2mo.cuh)


def flops(naux, nao, nocc, nvir):
    """Stage 1 per spin: 2 naux nao^2 na + 2 naux nao na nb (unpacked rows, smaller set na first, as ao2mo).  Pi per frequency:
    the executed tiles, T (T + 1) / 2 tiles of 64 x 64 with T = ceil(naux / 64), each 2 * 64 * 64 * K with K = sum nocc nvir."""
    f1 = 0.0
    for no, nv in zip(nocc, nvir):
        na, nb = min(no, nv), max(no, nv)
        f1 += 2.0 * naux * nao * nao * na + 2.0 * naux * nao * na * nb
    t = (naux + BM - 1) // BM
    k = sum(no * nv for no, nv in zip(nocc, nvir))
    return f1, t * (t + 1) / 2 * 2.0 * BM * BM * k


def torch_yardstick(naux, nov, reps=3):
    """ms of one frequency in torch fp64: (L chi) @ L^T with L [naux, nov] and cholesky(I - Pi), best of `reps` after a
    warm-up; the result is scaled by NW."""
    import torch
    g = torch.Generator(device='cuda').manual_seed(0)
    L = torch.randn(naux, nov, dtype=torch.float64, device='cuda', generator=g) * (0.3 / nov ** 0.5)
    chi = -torch.rand(nov, dtype=torch.float64, device='cuda', generator=g)
    eye = torch.eye(naux, dtype=torch.float64, device='cuda')
    best = {'gemm': None, 'cholesky': None}
    for i in range(reps + 1):
        ev = [torch.cuda.Event(enable_timing=True) for _ in range(3)]
        ev[0].record()
        pi = (L * chi) @ L.T
        ev[1].record()
        torch.linalg.cholesky(eye - pi)
        ev[2].record()
        ev[2].synchronize()
        if i:
            for k, (a, b) in zip(('gemm', 'cholesky'), ((0, 1), (1, 2))):
                t = ev[a].elapsed_time(ev[b])
                best[k] = t if best[k] is None else min(best[k], t)
    del L, chi, eye, pi
    torch.cuda.empty_cache()
    per = best['gemm'] + best['cholesky']
    return {'one_freq_gemm_ms': best['gemm'], 'one_freq_cholesky_ms': best['cholesky'], 'scaled_ms': per * NW,
            'gemm_TFLOPs_full_product': 2.0 * naux * naux * nov / (best['gemm'] * 1e-3) / 1e12}


def synthetic(nao, nocc, seed):
    rng = np.random.RandomState(seed)
    c = np.linalg.qr(rng.standard_normal((nao, nao)))[0]
    e = np.r_[np.sort(-1.0 - rng.random_sample(nocc)), np.sort(0.2 + rng.random_sample(nao - nocc))]
    return c, e


def run_case(d, label, cos, cvs, eos, evs, steps):
    from pyscf_b200 import rpa
    e_ovs = [(eo[:, None] - ev).ravel() for eo, ev in zip(eos, evs)]
    f_ovs = [np.full(x.size, 2.0 if len(cos) == 1 else 1.0) for x in e_ovs]
    call = lambda: rpa.kernel(d, cos, cvs, e_ovs, f_ovs, nw=NW)     # noqa: E731
    naux, nao = d.get_naoaux(), d.nao
    nocc = [c.shape[1] for c in cos]
    nvir = [c.shape[1] for c in cvs]
    f1, f2 = flops(naux, nao, nocc, nvir)
    e0 = call()          # warm-up: module load
    wall, st, es = [], [], []
    for _ in range(steps):
        t0 = time.perf_counter()
        es.append(call())
        wall.append(time.perf_counter() - t0)
        st.append(rpa.times(d))
    k = int(np.argsort(wall)[len(wall) // 2])
    t = st[k]
    return {'case': label, 'naux': naux, 'nao': nao, 'nocc': nocc, 'nvir': nvir, 'nw': NW, 'e_corr': es[k],
            'bitwise_repeatable': len(set(es + [e0])) == 1,
            'stage1_ms': t['stage1'], 'pi_ms': t['pi'], 'factor_ms': t['factor'],
            'stage1_TFLOP': f1 / 1e12, 'pi_TFLOP': NW * f2 / 1e12,
            'stage1_TFLOPs': f1 / (t['stage1'] * 1e-3) / 1e12 if t['stage1'] > 0 else None,
            'pi_TFLOPs': NW * f2 / (t['pi'] * 1e-3) / 1e12 if t['pi'] > 0 else None,
            'e2e_s': wall[k], 'e2e_s_all': wall,
            'device_share': (t['stage1'] + t['pi'] + t['factor']) * 1e-3 / wall[k]}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--steps', type=int, default=3)
    ap.add_argument('--only', default='bz_tz_rpa,c60_rpa,c60_urpa')
    ap.add_argument('--out', default=None)
    args = ap.parse_args()
    from pyscf_b200 import gto
    from pyscf_b200.df import DF
    from pyscf_b200.gto.mole import geometry
    only = args.only.split(',')
    res = {'card': card(), 'records': []}
    print(json.dumps(res['card']), flush=True)

    def emit(rec):
        res['records'].append(rec)
        print(json.dumps(rec), flush=True)

    if 'bz_tz_rpa' in only:
        mol = gto.M(atom=geometry('benzene'), basis='cc-pvtz')
        d = DF(mol).build()
        nocc = mol.nelectron // 2
        c, e = synthetic(d.nao, nocc, 1)
        rec = run_case(d, 'bz_tz_rpa', [c[:, :nocc]], [c[:, nocc:]], [e[:nocc]], [e[nocc:]], args.steps)
        rec['torch_yardstick'] = torch_yardstick(d.get_naoaux(), nocc * (d.nao - nocc))
        emit(rec)
        d.reset()
    if any(w.startswith('c60') for w in only):
        mol = gto.M(atom=geometry('c60'), basis='def2-svp')
        d = DF(mol).build()
        nocc = mol.nelectron // 2
        c, e = synthetic(d.nao, nocc, 2)
        naux, nvir = d.get_naoaux(), d.nao - nocc
        if 'c60_rpa' in only:
            rec = run_case(d, 'c60_rpa', [c[:, :nocc]], [c[:, nocc:]], [e[:nocc]], [e[nocc:]], args.steps)
            rec['torch_yardstick'] = torch_yardstick(naux, nocc * nvir)
            emit(rec)
        if 'c60_urpa' in only:
            cb, eb = synthetic(d.nao, nocc - 1, 3)
            rec = run_case(d, 'c60_urpa', [c[:, :nocc], cb[:, :nocc - 1]], [c[:, nocc:], cb[:, nocc - 1:]],
                           [e[:nocc], eb[:nocc - 1]], [e[nocc:], eb[nocc - 1:]], args.steps)
            rec['torch_yardstick'] = torch_yardstick(naux, nocc * nvir + (nocc - 1) * (nvir + 1))
            emit(rec)
        d.reset()
    if args.out:
        with open(args.out, 'w') as f:
            json.dump(res, f, indent=1)


if __name__ == '__main__':
    main()
