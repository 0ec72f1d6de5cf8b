#!/usr/bin/env python
"""Launch shape and time of every 4-center class of one direct J/K build: threads, dynamic shared memory, registers, spills,
CTAs per SM (occupancy API, under the carve-out the library sets, and from registers alone) and the class time (CUDA events
around each class launch, classes serialised, best of 3).  Prints a table; --json PATH also writes the record as JSON.
usage: python tools/occupancy_classes.py [--geom benzene --basis cc-pvtz] [--lib path/to/libb200jk.so] [--json out.json]"""
import argparse, ctypes, json, os, subprocess, sys
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import numpy as np
from pyscf_b200 import gto
from pyscf_b200.gto.mole import geometry
from pyscf_b200.jk import VHFOpt
from pyscf_b200 import lib as _lib

NAMES = ['ss', 'ps', 'pp', 'ds', 'dp', 'dd', 'fs', 'fp', 'fd', 'ff']
FIELDS = ['family', 'threads', 'smem', 'regs', 'local', 'ctas_sm', 'carveout', 'ctas_regs', 'swapped']


def card():
    import torch
    name = torch.cuda.get_device_name(0)
    try:   # read-only query
        power = subprocess.run(['nvidia-smi', '--query-gpu=power.limit', '--format=csv,noheader', '-i', '0'],
                               capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception as e:
        power = 'unknown (%s)' % e
    return name, power


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--geom', default='benzene')
    ap.add_argument('--basis', default='cc-pvtz')
    ap.add_argument('--nocc', type=int, default=21)
    ap.add_argument('--lib', default=None)
    ap.add_argument('--json', default=None, help='also write the record to this JSON file')
    a = ap.parse_args()
    mol = gto.M(atom=geometry(a.geom), basis=a.basis)
    c, _ = np.linalg.qr(np.random.RandomState(1).standard_normal((mol.nao, a.nocc)))
    dm = 2 * c.dot(c.T)
    opt = VHFOpt(mol, libpath=os.path.abspath(a.lib) if a.lib else None)
    h = opt.handle
    info_fn = h.lib.b200jk_class_launch_info
    info_fn.argtypes = [ctypes.c_void_p, ctypes.c_int, ctypes.c_int, ctypes.POINTER(ctypes.c_int), ctypes.c_int]
    for _ in range(3):
        opt.get_jk(dm)
    ms = []
    for _ in range(5):
        opt.get_jk(dm)
        ms.append(opt.stats()['ms_kernels'])
    h.lib.b200jk_set_profile(h._h, 1)
    best = None
    for _ in range(3):
        opt.get_jk(dm)
        cm = np.zeros(100)
        h.lib.b200jk_get_class_times(h._h, _lib.dptr(cm), 100)
        best = cm if best is None else np.minimum(best, cm)
    name, power = card()
    rows = {}
    for cb in range(10):
        for ck in range(cb + 1):
            if not best[cb * 10 + ck] > 0:
                continue
            buf = (ctypes.c_int * 9)()
            if info_fn(h._h, cb, ck, buf, 9) != 0:
                raise RuntimeError(h.lib.b200jk_last_error(h._h).decode())
            r = dict(zip(FIELDS, list(buf)))
            r['ms'] = float(best[cb * 10 + ck])
            rows['(%s|%s)' % (NAMES[cb], NAMES[ck])] = r
    out = {'card': name, 'power_limit': power, 'lib': a.lib or _lib.DEFAULT_LIB, 'build_ms_best': min(ms),
           'build_ms_mean': float(np.mean(ms)), 'class_ms_sum': float(best.sum()), 'classes': rows}
    print('%s, power limit %s; build %.3f ms best / %.3f ms mean (unprofiled), class sum %.3f ms (profiled)'
          % (name, power, min(ms), np.mean(ms), best.sum()))
    print('%-9s %-5s %4s %7s %4s %5s %5s %5s %5s %8s' % ('class', 'fam', 'thr', 'smem', 'reg', 'local', 'carve', 'cta', 'ctaR', 'ms'))
    for k, r in sorted(rows.items(), key=lambda kv: -kv[1]['ms']):
        print('%-9s %-5s %4d %7d %4d %5d %5d %5d %5d %8.3f%s' % (k, ('tpq', 'block', 'swq')[r['family']], r['threads'], r['smem'],
              r['regs'], r['local'], r['carveout'], r['ctas_sm'], r['ctas_regs'], r['ms'], ' swapped' if r['swapped'] else ''))
    if a.json:
        d = os.path.dirname(os.path.abspath(a.json))
        os.makedirs(d, exist_ok=True)
        with open(a.json, 'w') as f:
            json.dump(out, f, indent=1)
    opt.close()


if __name__ == '__main__':
    main()
