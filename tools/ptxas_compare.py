#!/usr/bin/env python
"""Compare registers / spills per kernel between two sets of `ptxas -v` logs (e.g. pyscf_b200/csrc/build/ptxas_bra_*.log and
/tmp/b200jk_variant_<name>/obj/ptxas_*.log).  usage: python tools/ptxas_compare.py 'globA' 'globB'"""
import glob, re, sys


def parse(pattern):
    out = {}
    for f in glob.glob(pattern):
        txt = open(f).read()
        for m in re.finditer(r"Compiling entry function '(\S+)' for 'sm_90a'.*?(\d+) bytes stack frame, (\d+) bytes spill stores.*?Used (\d+) registers", txt, re.S):
            mm = re.search(r'jk_(class_kernel_2cta|class_kernel|tpq_kernel)INS_6QClassILi(\d)ELi(\d)ELi(\d)ELi(\d)ELi(\d+)E(?:Li(\d+)E)?EELb(\d)', m.group(1))
            if mm and mm.group(8) == '0':
                key = '(%s%s|%s%s)' % tuple('spdfg'[int(x)] for x in mm.group(2, 3, 4, 5))
                out[key] = (mm.group(1).replace('class_kernel', 'blk').replace('_kernel', ''), int(mm.group(6)), int(mm.group(7) or 1),
                            int(m.group(4)), int(m.group(3)))
    return out


a, b = parse(sys.argv[1]), parse(sys.argv[2])
print('%-9s %-9s %3s %3s %5s %6s   ->  %-9s %3s %3s %5s %6s' % ('class', 'kernel', 'NP', 'PB', 'regs', 'spill', 'kernel', 'NP', 'PB', 'regs', 'spill'))
for k in sorted(a):
    if k in b and a[k] != b[k]:
        print('%-9s %-9s %3d %3d %5d %6d   ->  %-9s %3d %3d %5d %6d' % ((k,) + a[k] + b[k]))
