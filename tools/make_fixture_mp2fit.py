#!/usr/bin/env python
"""Freeze the H and O shells of the cc-pVDZ-RI auxiliary basis (the MP2-fit basis make_auxbasis(mol, mp2fit=True) picks for
cc-pVDZ, pyscf/df/addons.py:42-72) as tests/golden/basis_cc-pvdz-ri.json, a test fixture of tests/test_df_mp2.py.

Needs a checkout of the reference at REF; the output is committed, so the tests never read it.  Source: pyscf/gto/basis/cc-pvdz-ri.dat
(NWChem format), parsed with this repository's parser (pyscf_b200.gto.basis.parse_nwchem) as tools/make_fixtures.py does."""
import json
import os
import sys

REF = '/root/reference'
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from pyscf_b200.gto.basis import parse_nwchem, extract_element_block


def main():
    text = open(os.path.join(REF, 'pyscf/gto/basis/cc-pvdz-ri.dat')).read()
    out = {el: parse_nwchem(extract_element_block(text, el)) for el in ('H', 'O')}
    path = os.path.join(ROOT, 'tests', 'golden', 'basis_cc-pvdz-ri.json')
    with open(path, 'w') as f:
        json.dump(out, f, separators=(',', ':'))
    print(path, {k: len(v) for k, v in out.items()})


if __name__ == '__main__':
    main()
