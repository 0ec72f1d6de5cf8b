"""Measure DF-MP2 on one GPU (pyscf_b200.dfmp2: b200jk_df_mp2, df_mp2.cuh).

Workloads (random orthonormal orbitals and synthetic energies, occupied < 0 < virtual: the time does not depend on the values):
  bz_tz_rmp2   benzene/cc-pVTZ, full RMP2
  c60_rmp2     C60/def2-SVP, full RMP2 (nocc 180, nvir 660, naux 4500: 63.9 TFLOP in stage 2), with_t2=False (t2 would be 113 GB)
  c60_ump2     C60/def2-SVP, UMP2 with nocc_beta = nocc_alpha - 1
Per workload: the card name and power limit (read in the same process), stage-1 and stage-2 device time (CUDA events inside the
library), the FLOPs of each stage counted here from the shapes, the achieved FP64 TFLOP/s, and the end-to-end wall time of the
call (median of `--steps` after one warm-up call), with the share of that time the two stages take.
Yardsticks in the same process:
  * the route through DF.ao2mo: (ia|jb) to the host, then the energy in numpy, for benzene and for a 20-orbital occupied window
    of C60 (the DF-MP2 kernel runs on the same window: the parity of the two energies is reported);
  * cuBLAS: torch.bmm in fp64 on batches of [nvir, naux] x [naux, nvir], the product of one pair, scaled to all pairs.

    python tools/bench_df_mp2.py [--steps 3] [--only bz_tz_rmp2,c60_rmp2,c60_ump2] [--out FILE]
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


def flops(naux, nao, nocc, nvir):
    """Stage 1 per spin: 2 naux nao^2 na + 2 naux nao na nb (unpacked rows, smaller set na first, as ao2mo).  Stage 2: the full
    V = L_i^T L_j of every pair, 2 nvir_a nvir_b naux per pair, over i >= j pairs per spin and all alpha-beta pairs."""
    f1 = f2 = 0.0
    for no, nv in zip(nocc, nvir):
        na, nb = min(no, nv), max(no, nv)
        f1 += 2.0 * naux * nao * nao * na + 2.0 * naux * nao * na * nb
        f2 += no * (no + 1) / 2 * 2.0 * nv * nv * naux
    if len(nocc) == 2:
        f2 += nocc[0] * nocc[1] * 2.0 * nvir[0] * nvir[1] * naux
    return f1, f2


def npairs(nocc):
    n = sum(no * (no + 1) // 2 for no in nocc)
    return n + (nocc[0] * nocc[1] if len(nocc) == 2 else 0)


def cublas_yardstick(naux, nvir, pairs, batch=32, reps=3):
    """ms of torch.bmm on `batch` pairs of [nvir, naux] x [naux, nvir] in fp64 (cuBLAS), best of `reps` after a warm-up, scaled
    to `pairs` pairs."""
    import torch
    a = torch.randn(batch, nvir, naux, dtype=torch.float64, device='cuda')
    b = torch.randn(batch, naux, nvir, dtype=torch.float64, device='cuda')
    c = torch.empty(batch, nvir, nvir, dtype=torch.float64, device='cuda')
    best = None
    for i in range(reps + 1):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        torch.bmm(a, b, out=c)
        e1.record()
        e1.synchronize()
        if i:
            t = e0.elapsed_time(e1)
            best = t if best is None else min(best, t)
    del a, b, c
    torch.cuda.empty_cache()
    ms = best * pairs / batch
    return {'batch': batch, 'batch_ms': best, 'scaled_ms': ms, 'TFLOPs': 2.0 * nvir * nvir * naux * pairs / (ms * 1e-3) / 1e12}


def numpy_energy(ovov, eo, ev):
    """RMP2 (e_ss, e_os) from (ia|jb) [nocc nvir, nocc nvir] on the host (mp2.py:808-830 reshaped pair by pair)."""
    no, nv = len(eo), len(ev)
    ed = ex = 0.0
    for i in range(no):
        g = ovov[i * nv:(i + 1) * nv].reshape(nv, no, nv).transpose(1, 0, 2)
        t = g / (eo[i] + eo[:, None, None] - ev[None, :, None] - ev[None, None, :])
        ed += np.einsum('jab,jab', t, g)
        ex -= np.einsum('jab,jba', t, g)
    return ed + ex, ed


def ao2mo_route(d, co, cv, eo, ev):
    """The route through DF.ao2mo: (ia|jb) to the host, then the numpy energy; seconds of each and the energy."""
    t0 = time.perf_counter()
    ovov = d.ao2mo((co, cv, co, cv))
    t1 = time.perf_counter()
    e_ss, e_os = numpy_energy(ovov, eo, ev)
    t2 = time.perf_counter()
    return {'ao2mo_s': t1 - t0, 'numpy_energy_s': t2 - t1, 'total_s': t2 - t0, 'ovov_GB': ovov.nbytes / 1e9,
            'e_corr': e_ss + e_os, 'e_ss': e_ss, 'e_os': e_os}


def synthetic(nao, nocc, seed):
    rng = np.random.RandomState(seed)
    c = np.linalg.qr(rng.standard_normal((nao, nao)))[0]
    e = np.r_[np.sort(-1.0 - rng.random_sample(nocc)), np.sort(0.2 + rng.random_sample(nao - nocc))]
    return c, e


def run_case(d, label, cos, cvs, eos, evs, steps, with_t2=False):
    from pyscf_b200 import dfmp2
    unrestricted = len(cos) == 2
    call = (lambda: dfmp2.ukernel(d, cos, cvs, eos, evs, with_t2)) if unrestricted else \
        (lambda: dfmp2.kernel(d, cos[0], cvs[0], eos[0], evs[0], with_t2))
    naux, nao = d.get_naoaux(), d.nao
    nocc = [c.shape[1] for c in cos]
    nvir = [c.shape[1] for c in cvs]
    f1, f2 = flops(naux, nao, nocc, nvir)
    e = call()[0]          # warm-up: module load, shared-memory attribute
    wall, st, es = [], [], []
    for _ in range(steps):
        t0 = time.perf_counter()
        r = call()
        wall.append(time.perf_counter() - t0)
        st.append(dfmp2.times(d))
        es.append((float(r[0]), r[0].e_corr_ss, r[0].e_corr_os))
        del r
    k = int(np.argsort(wall)[len(wall) // 2])
    t = st[k]
    dev_s = (t['stage1'] + t['stage2']) * 1e-3
    return {'case': label, 'naux': naux, 'nao': nao, 'nocc': nocc, 'nvir': nvir, 'with_t2': with_t2,
            'e_corr': es[k][0], 'e_ss': es[k][1], 'e_os': es[k][2], 'bitwise_repeatable': len(set(es + [(float(e), e.e_corr_ss,
                                                                                                         e.e_corr_os)])) == 1,
            'stage1_ms': t['stage1'], 'stage2_ms': t['stage2'], 'stage1_TFLOP': f1 / 1e12, 'stage2_TFLOP': f2 / 1e12,
            'stage1_TFLOPs': f1 / (t['stage1'] * 1e-3) / 1e12 if t['stage1'] > 0 else None,
            'stage2_TFLOPs': f2 / (t['stage2'] * 1e-3) / 1e12 if t['stage2'] > 0 else None,
            'e2e_s': wall[k], 'e2e_s_all': wall,
            'bound': 'device compute: the two stages take %.0f %% of the call' % (100 * dev_s / wall[k]) if dev_s > 0.6 * wall[k]
                     else 'host side: the two stages take %.0f %% of the call' % (100 * dev_s / wall[k])}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--steps', type=int, default=3)
    ap.add_argument('--only', default='bz_tz_rmp2,c60_rmp2,c60_ump2')
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

    if 'bz_tz_rmp2' in only:
        mol = gto.M(atom=geometry('benzene'), basis='cc-pvtz')
        d = DF(mol).build()
        nocc = mol.nelectron // 2
        c, e = synthetic(d.nao, nocc, 1)
        co, cv, eo, ev = c[:, :nocc], c[:, nocc:], e[:nocc], e[nocc:]
        rec = run_case(d, 'bz_tz_rmp2', [co], [cv], [eo], [ev], args.steps)
        rec['with_t2_e2e_s'] = run_case(d, 'bz_tz_rmp2 t2', [co], [cv], [eo], [ev], 1, with_t2=True)['e2e_s']
        rec['ao2mo_route'] = ao2mo_route(d, co, cv, eo, ev)
        rec['ao2mo_route']['abs_diff_e_corr'] = abs(rec['ao2mo_route']['e_corr'] - rec['e_corr'])
        rec['cublas_bmm'] = cublas_yardstick(d.get_naoaux(), cv.shape[1], npairs([nocc]))
        emit(rec)
        d.reset()
    if any(w.startswith('c60') for w in only):
        mol = gto.M(atom=geometry('c60'), basis='def2-svp')
        d = DF(mol).build()
        nocc = mol.nelectron // 2
        c, e = synthetic(d.nao, nocc, 2)
        co, cv, eo, ev = c[:, :nocc], c[:, nocc:], e[:nocc], e[nocc:]
        naux, nvir = d.get_naoaux(), cv.shape[1]
        if 'c60_rmp2' in only:
            rec = run_case(d, 'c60_rmp2', [co], [cv], [eo], [ev], args.steps)
            rec['cublas_bmm'] = cublas_yardstick(naux, nvir, npairs([nocc]))
            emit(rec)
            # the 20-orbital window: the kernel against the DF.ao2mo route
            w = slice(nocc - 20, nocc)
            win = run_case(d, 'c60_window20_rmp2', [co[:, w]], [cv], [eo[w]], [ev], args.steps)
            win['ao2mo_route'] = ao2mo_route(d, co[:, w], cv, eo[w], ev)
            win['ao2mo_route']['abs_diff_e_corr'] = abs(win['ao2mo_route']['e_corr'] - win['e_corr'])
            win['ao2mo_route']['abs_diff_e_ss'] = abs(win['ao2mo_route']['e_ss'] - win['e_ss'])
            win['ao2mo_route']['abs_diff_e_os'] = abs(win['ao2mo_route']['e_os'] - win['e_os'])
            emit(win)
        if 'c60_ump2' in only:
            cb, eb = synthetic(d.nao, nocc - 1, 3)
            rec = run_case(d, 'c60_ump2', [co, cb[:, :nocc - 1]], [cv, cb[:, nocc - 1:]], [eo, eb[:nocc - 1]], [ev, eb[nocc - 1:]],
                           args.steps)
            rec['cublas_bmm'] = cublas_yardstick(naux, nvir, npairs([nocc, nocc - 1]))
            emit(rec)
        d.reset()
    if args.out:
        with open(args.out, 'w') as f:
            json.dump(res, f, indent=1)


if __name__ == '__main__':
    main()
