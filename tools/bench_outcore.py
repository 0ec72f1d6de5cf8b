"""Measure DF J/K with tensor rows streamed from pinned host memory (b200jk_df_set_device_rows) on one GPU.

Reports, in one run: the card and its power limit; the pinned host -> device bandwidth of one large copy timed with CUDA
events; C60/def2-SVP per-build time with 0 %, 50 % and 100 % of the rows forced to the host against the all-resident build
(variants alternated, each rebuilt per round); Taxol/def2-TZVP with the automatic split: setup time, per-build time, host
bytes per build, copy time and the copy time the compute stream waited for.

    python tools/bench_outcore.py [--rounds 2] [--steps 3] [--no-taxol] [--out FILE]
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def card():
    import torch
    name = torch.cuda.get_device_name(0)
    try:
        out = subprocess.run(['nvidia-smi', '--query-gpu=power.limit', '--format=csv,noheader,nounits', '-i', '0'],
                             capture_output=True, text=True, timeout=30).stdout.strip()
        power = float(out.splitlines()[0])
    except Exception:
        power = None
    return {'gpu': name, 'power_limit_w': power}


def h2d_bandwidth(nbytes=4 << 30, reps=3):
    """GB/s of one pinned host -> device copy of `nbytes`, best of `reps`, CUDA events around the copy."""
    import torch
    src = torch.empty(nbytes, dtype=torch.uint8, pin_memory=True)
    dst = torch.empty(nbytes, dtype=torch.uint8, device='cuda')
    best = 0.0
    for _ in range(reps + 1):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        dst.copy_(src, non_blocking=True)
        b.record()
        b.synchronize()
        best = max(best, nbytes / (a.elapsed_time(b) * 1e-3) / 1e9)
    del src, dst
    torch.cuda.empty_cache()
    return best


def scf_like_density(nao, nocc, seed=1):
    from pyscf_b200.df import TaggedDM
    co, _ = np.linalg.qr(np.random.RandomState(seed).standard_normal((nao, nocc)))
    return TaggedDM(2.0 * co.dot(co.T), mo_coeff=co, mo_occ=np.full(nocc, 2.0))


def time_builds(d, dm, steps):
    """Wall-clock ms per J/K build (median of `steps` after one warm-up) and the stream statistics of the last build."""
    d.get_jk(dm, hermi=1)
    t = []
    for _ in range(steps):
        t0 = time.perf_counter()
        d.get_jk(dm, hermi=1)
        t.append((time.perf_counter() - t0) * 1e3)
    return float(np.median(t)), d.stream_stats()


def c60(rounds, steps):
    from pyscf_b200 import gto
    from pyscf_b200.df import DF
    from pyscf_b200.gto.mole import geometry
    mol = gto.M(atom=geometry('c60'), basis='def2-svp')
    dm = scf_like_density(mol.nao, mol.nelectron // 2)
    d = DF(mol).build()
    naux = d.get_naoaux()
    d.reset()
    variants = {'resident': -1, 'host_0pct': naux, 'host_50pct': naux - naux // 2, 'host_100pct': 0}
    res = {k: [] for k in variants}
    for r in range(rounds):
        for name, cap in (variants.items() if r % 2 == 0 else reversed(list(variants.items()))):
            d = DF(mol).set_device_rows(cap).build()
            ms, st = time_builds(d, dm, steps)
            res[name].append({'ms': ms, 'split': d.row_split(), **st})
            d.reset()
    return {'naux': naux, 'nao': mol.nao, 'variants': res}


def taxol(steps):
    from pyscf_b200 import gto
    from pyscf_b200.df import DF
    from pyscf_b200.gto.mole import geometry
    mol = gto.M(atom=geometry('taxol'), basis='def2-tzvp')
    t0 = time.perf_counter()
    d = DF(mol).build()
    setup_s = time.perf_counter() - t0
    dm = scf_like_density(mol.nao, mol.nelectron // 2)
    ms, st = time_builds(d, dm, steps)
    out = {'setup_s': setup_s, 'ms': ms, 'split': d.row_split(), **st, 'stage_times': d.stage_times()}
    d.reset()
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--rounds', type=int, default=2)
    ap.add_argument('--steps', type=int, default=3)
    ap.add_argument('--no-taxol', action='store_true')
    ap.add_argument('--out', default=None)
    a = ap.parse_args()
    rec = card()
    rec['h2d_pinned_GBps'] = h2d_bandwidth()
    print(json.dumps(rec), flush=True)
    rec['c60_def2svp'] = c60(a.rounds, a.steps)
    print(json.dumps({'c60_def2svp': rec['c60_def2svp']}), flush=True)
    if not a.no_taxol:
        rec['taxol_def2tzvp'] = taxol(a.steps)
        print(json.dumps({'taxol_def2tzvp': rec['taxol_def2tzvp']}), flush=True)
    if a.out:
        with open(a.out, 'w') as f:
            json.dump(rec, f, indent=1)


if __name__ == '__main__':
    main()
