"""Measure DF.ao2mo (MO integrals from the fitted tensor, df_ao2mo.cuh) on one GPU.

Workloads, the shapes post-SCF codes hand to with_df.ao2mo:
  c60_cas16   C60/def2-SVP, 16 active orbitals: paaa = ao2mo([mo, cas, cas, cas], compact=False) then aaaa = ao2mo(cas)
              (one DF-CASSCF macro iteration, pyscf/mcscf/df.py:140,160)
  c60_ovov60  C60/def2-SVP, (ia|jb) over 60 occupied x all virtual orbitals (12.5 GB output: several output bands)
  bz_tz_ovov  benzene/cc-pVTZ, full (ia|jb) (mp.MP2, pyscf/mp/mp2.py:808-814)
Per workload: the card name and power limit (read in the same process), stage-1 and stage-2 device time (CUDA events inside the
library), the FLOPs each stage executes (counted here from the shapes) and the achieved FP64 TFLOP/s, the end-to-end wall time
of the call including the device-to-host copy into the caller's array (median of `--steps` after one warm-up call) and which
bound holds.  Yardsticks: torch.matmul in fp64 (cuBLAS) on random matrices of the shapes of L and L' (a dense GEMM's time does
not depend on the values), and numpy on the CPU for a sample of tensor rows, scaled to all rows.

    python tools/bench_df_ao2mo.py [--steps 3] [--only c60_cas16,c60_ovov60,bz_tz_ovov] [--out FILE]
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

BAND_BYTES = 256 << 20     # output band of df_ao2mo.cuh (ao2mo_band_rows)


def flops(naux, nao, sets, s12, s34, sym):
    """FLOPs the library executes: stage 1 per pair 2 naux nao^2 na + 2 naux nao na nb (unpacked rows, smaller set na first;
    s2 pairs still form the whole na x nb block), stage 2 2 naux nij nkl, less the mirrored upper triangles of the diagonal
    blocks of the output bands when pair (3,4) is pair (1,2) (tile granularity ignored)."""
    def pair(n1, n2):
        na, nb = min(n1, n2), max(n1, n2)
        return 2.0 * naux * nao * nao * na + 2.0 * naux * nao * na * nb
    n = sets
    nij = n[0] * (n[0] + 1) // 2 if s12 else n[0] * n[1]
    nkl = n[2] * (n[2] + 1) // 2 if s34 else n[2] * n[3]
    f1 = pair(n[0], n[1]) + (0.0 if sym else pair(n[2], n[3]))
    if sym:
        band = max(1, min(nij, BAND_BYTES // (nkl * 8)))
        cells = 0
        for r0 in range(0, nij, band):
            r = min(band, nij - r0)
            cells += r * nkl - r * (r - 1) // 2
        f2 = 2.0 * naux * cells
    else:
        f2 = 2.0 * naux * nij * nkl
    return f1, f2, nij, nkl


def torch_yardstick(naux, nij, nkl, sym, reps=3):
    """ms of torch.matmul(L^T, L') in fp64 on the GPU (cuBLAS DGEMM), best of `reps` after a warm-up; None if it does not fit."""
    import torch
    try:
        a = torch.randn(naux, nij, dtype=torch.float64, device='cuda')
        b = a if sym else torch.randn(naux, nkl, dtype=torch.float64, device='cuda')
        c = torch.empty(nij, nkl, dtype=torch.float64, device='cuda')
    except RuntimeError:
        torch.cuda.empty_cache()
        return None
    best = None
    for i in range(reps + 1):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        torch.matmul(a.t(), b, out=c)
        e1.record()
        e1.synchronize()
        if i:
            t = e0.elapsed_time(e1)
            best = t if best is None else min(best, t)
    del a, b, c
    torch.cuda.empty_cache()
    return best


def numpy_sample(d, cs, s12, s34, sym, rows=32):
    """CPU seconds of the numpy transform (unpack, half transforms, output GEMM) of `rows` tensor rows, and that time scaled to
    all rows (the transform is linear in the row count)."""
    nao = d.nao
    blk = next(d.loop(blksize=rows))
    t0 = time.perf_counter()
    Bf = np.zeros((len(blk), nao, nao))
    i, j = np.tril_indices(nao)
    Bf[:, i, j] = blk
    Bf[:, j, i] = blk

    def half(c1, c2, s2):
        L = np.einsum('pmn,mi,nj->pij', Bf, c1, c2, optimize=True)
        if s2:
            a, b = np.tril_indices(c1.shape[1])
            return L[:, a, b]
        return L.reshape(len(Bf), -1)
    L1 = half(cs[0], cs[1], s12)
    L2 = L1 if sym else half(cs[2], cs[3], s34)
    L1.T @ L2
    t = time.perf_counter() - t0
    return {'rows': len(blk), 'seconds': t, 'scaled_to_all_rows_s': t * d.get_naoaux() / len(blk)}


def run_case(d, label, cs, compact, steps):
    from pyscf_b200.df import _iden_coeffs
    four = (cs,) * 4 if isinstance(cs, np.ndarray) else cs
    n = [c.shape[1] for c in four]
    s12 = bool(compact and _iden_coeffs(four[0], four[1]))
    s34 = bool(compact and _iden_coeffs(four[2], four[3]))
    sym = bool(s12 == s34 and _iden_coeffs(four[0], four[2]) and _iden_coeffs(four[1], four[3]))
    naux, nao = d.get_naoaux(), d.nao
    f1, f2, nij, nkl = flops(naux, nao, n, s12, s34, sym)
    d.ao2mo(cs, compact=compact)          # warm-up: module load, pinned staging
    wall, st = [], []
    for _ in range(steps):
        t0 = time.perf_counter()
        out = d.ao2mo(cs, compact=compact)
        wall.append(time.perf_counter() - t0)
        st.append(d.ao2mo_times())
        del out
    k = int(np.argsort(wall)[len(wall) // 2])
    t = st[k]
    out_gb = nij * nkl * 8 / 1e9
    e2e = wall[k]
    dev_s = (t['stage1'] + t['stage2']) * 1e-3
    rec = {'case': label, 'naux': naux, 'nao': nao, 'sets': n, 's12': s12, 's34': s34, 'sym': sym, 'nij': nij, 'nkl': nkl,
           'out_GB': out_gb, 'stage1_ms': t['stage1'], 'stage2_ms': t['stage2'],
           'stage1_GFLOP': f1 / 1e9, 'stage2_GFLOP': f2 / 1e9,
           'stage1_TFLOPs': f1 / (t['stage1'] * 1e-3) / 1e12 if t['stage1'] > 0 else None,
           'stage2_TFLOPs': f2 / (t['stage2'] * 1e-3) / 1e12 if t['stage2'] > 0 else None,
           'e2e_s': e2e, 'e2e_s_all': wall, 'e2e_output_GBps': out_gb / e2e,
           'bound': 'device compute (stage kernels %.0f %% of the call)' % (100 * dev_s / e2e) if dev_s > 0.6 * e2e else
                    'copies to the caller (stage kernels %.0f %% of the call)' % (100 * dev_s / e2e)}
    rec['torch_fp64_matmul_ms'] = torch_yardstick(naux, nij, nkl, sym)
    if rec['torch_fp64_matmul_ms']:
        rec['torch_fp64_matmul_TFLOPs'] = 2.0 * naux * nij * nkl / (rec['torch_fp64_matmul_ms'] * 1e-3) / 1e12
    rec['numpy_cpu'] = numpy_sample(d, list(four), s12, s34, sym)
    return rec


def orbitals(nao, seed):
    return np.linalg.qr(np.random.RandomState(seed).standard_normal((nao, nao)))[0]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--steps', type=int, default=3)
    ap.add_argument('--only', default='c60_cas16,c60_ovov60,bz_tz_ovov')
    ap.add_argument('--out', default=None)
    args = ap.parse_args()
    from pyscf_b200 import gto
    from pyscf_b200.df import DF
    from pyscf_b200.gto.mole import geometry
    only = args.only.split(',')
    res = {'card': card(), 'records': []}
    print(json.dumps(res['card']), flush=True)
    if any(w.startswith('c60') for w in only):
        mol = gto.M(atom=geometry('c60'), basis='def2-svp')
        d = DF(mol).build()
        mo = orbitals(d.nao, 1)
        nocc = mol.nelectron // 2
        if 'c60_cas16' in only:
            cas = mo[:, nocc - 8:nocc + 8]
            for label, cs, compact in (('c60_cas16 paaa', [mo, cas, cas, cas], False), ('c60_cas16 aaaa', cas, True)):
                res['records'].append(run_case(d, label, cs, compact, args.steps))
                print(json.dumps(res['records'][-1]), flush=True)
        if 'c60_ovov60' in only:
            co, cv = mo[:, nocc - 60:nocc], mo[:, nocc:]
            res['records'].append(run_case(d, 'c60_ovov60', (co, cv, co, cv), True, args.steps))
            print(json.dumps(res['records'][-1]), flush=True)
        d.reset()
    if 'bz_tz_ovov' in only:
        mol = gto.M(atom=geometry('benzene'), basis='cc-pvtz')
        d = DF(mol).build()
        mo = orbitals(d.nao, 2)
        nocc = mol.nelectron // 2
        res['records'].append(run_case(d, 'bz_tz_ovov', (mo[:, :nocc], mo[:, nocc:], mo[:, :nocc], mo[:, nocc:]), True,
                                       args.steps))
        print(json.dumps(res['records'][-1]), flush=True)
        d.reset()
    if args.out:
        with open(args.out, 'w') as f:
            json.dump(res, f, indent=1)


if __name__ == '__main__':
    main()
