"""Density-fitting tensors larger than the device: the rows that do not fit stay in pinned host memory and are streamed through
two device staging buffers once per J/K call (b200jk_df_set_device_rows / b200jk_df_row_split / b200jk_df_stream_stats).

CPU emulation (the "pinned" buffer is plain host memory; the split, blocking and staging logic is the same code): H2O/cc-pVDZ
and He-Ne/cc-pVTZ with forced device rows against the all-resident handle and the oracle.  GPU: C60/def2-SVP with forced
splits against the size fixture and the all-resident build, Taxol/def2-TZVP with the automatic split on one GPU, and the
automatic split leaving tensors that fit entirely on the device."""
import os
import subprocess
import sys

import numpy as np
import pytest

from pyscf_b200 import gto
from pyscf_b200.df import DF, TaggedDM
from pyscf_b200.gto.mole import geometry, make_auxmol
from oracle import oracle as O

CASES = {'h2o': ('O 0 0 0; H 0 -0.757 0.587; H 0 0.757 0.587', 'cc-pvdz', 'weigend'),
         'hene': ('He 0 0 0; Ne 1.2 0.3 0', 'cc-pvtz', 'def2-universal-jkfit')}


def _set_kblock(d, kb):
    h = d._handle
    h.check(h.lib.b200jk_df_set_kblock(h._h, int(kb), -1), 'b200jk_df_set_kblock')


def _inputs(nao, seed=1):
    """Two orbital-tagged densities (K through the occupied-orbital algorithm, one orbital set per call) and two general
    densities with hermi 0 and 1 (n_dm = 2 in one call)."""
    rng = np.random.RandomState(seed)
    c1, c2 = (np.linalg.qr(rng.standard_normal((nao, 4)))[0] * np.sqrt(2.0) for _ in range(2))
    dm_g = rng.random_sample((2, nao, nao))
    dm_s = dm_g + dm_g.transpose(0, 2, 1)
    dms_t = np.array([c1 @ c1.T, c2 @ c2.T])
    return {'tagged': (TaggedDM(dms_t, mo_coeff=np.array([c1, c2]), mo_occ=np.full((2, 4), 1.0)), 1, dms_t),
            'general0': (dm_g, 0, dm_g), 'general1': (dm_s, 1, dm_s)}


def _emu_case(name, emu_lib):
    atom, basis, aux = CASES[name]
    mol = gto.M(atom=atom, basis=basis)
    ref, nao = O.cholesky_eri(mol, make_auxmol(mol, aux))
    d0 = DF(mol, aux, libpath=emu_lib).build()
    return mol, aux, ref, nao, d0


@pytest.mark.parametrize('name', ['h2o', 'hene'])
def test_split_jk_emulated(emu_lib, name):
    """Forced device rows 0, 1, naux/3 and naux - 1 with K blocks of a few rows (several staged blocks per call) against the
    all-resident handle (1e-12) and the oracle (1e-9): tagged and general densities, hermi 0 and 1, n_dm = 2."""
    mol, aux, ref, nao, d0 = _emu_case(name, emu_lib)
    naux = d0.get_naoaux()
    npair = nao * (nao + 1) // 2
    assert d0.row_split() == (naux, 0)
    inputs = _inputs(nao)
    want = {k: d0.get_jk(v[0], hermi=v[1]) for k, v in inputs.items()}
    assert d0.stream_stats()['bytes'] == 0
    for kind, (_, _, dms) in inputs.items():
        rj, rk = O.df_get_jk(ref, nao, dms)
        assert abs(want[kind][0] - rj).max() < 1e-9 and abs(want[kind][1] - rk).max() < 1e-9, kind
    for cap in (0, 1, naux // 3, naux - 1):
        d = DF(mol, aux, libpath=emu_lib).set_device_rows(cap).build()
        assert d.row_split() == (cap, naux - cap)
        _set_kblock(d, max(1, (naux - cap) // 7))
        for kind, (dm, hermi, dms) in inputs.items():
            vj, vk = d.get_jk(dm, hermi=hermi)
            assert abs(vj - want[kind][0]).max() < 1e-12 and abs(vk - want[kind][1]).max() < 1e-12, (cap, kind)
            rj, rk = O.df_get_jk(ref, nao, dms)
            assert abs(vj - rj).max() < 1e-9 and abs(vk - rk).max() < 1e-9, (cap, kind)
        # the last call (general density, J and K) crossed each host row once
        assert d.stream_stats()['bytes'] == (naux - cap) * npair * 8
        vj, _ = d.get_jk(inputs['general1'][0], hermi=1, with_k=False)          # J alone on staged rows
        assert abs(vj - want['general1'][0]).max() < 1e-12
        _, vk = d.get_jk(inputs['general1'][0], hermi=1, with_j=False)          # K alone
        assert abs(vk - want['general1'][1]).max() < 1e-12


def test_split_tensor_access_emulated(emu_lib, tmp_path):
    """loop(), cderi_columns() and save() with a split return the resident tensor bit for bit; an assigned tensor (_cderi,
    set_cderi) is split as well and gives the same J/K."""
    mol, aux, ref, nao, d0 = _emu_case('h2o', emu_lib)
    naux = d0.get_naoaux()
    full = d0._cderi
    cols = np.array([0, 1, 5, 17, nao * (nao + 1) // 2 - 1])
    for cap in (0, naux // 3, naux - 1):
        d = DF(mol, aux, libpath=emu_lib).set_device_rows(cap).build()
        blocks = list(d.loop(blksize=7))
        assert np.array_equal(np.vstack(blocks), full)
        assert np.array_equal(d.cderi_columns(cols), full[:, cols])
        path = d.save(str(tmp_path / ('cderi_%d.npy' % cap)))
        assert np.array_equal(np.load(path), full)
        # assigned tensor, split at another row
        d2 = DF(mol, aux, libpath=emu_lib).set_device_rows(naux - 1 - cap)
        d2._cderi = full
        dm = _inputs(nao)['general1'][0]
        vj, vk = d2.get_jk(dm, hermi=1)
        assert d2.row_split() == (naux - 1 - cap, cap + 1)
        wj, wk = d0.get_jk(dm, hermi=1)
        assert abs(vj - wj).max() < 1e-12 and abs(vk - wk).max() < 1e-12
        assert np.array_equal(d2._cderi, full)


def test_split_sharded_emulated(emu_lib):
    """Two ranks, each holding half of the rows and keeping only a few of them on the device: the partial J/K sum to the
    full result."""
    mol, aux, ref, nao, d0 = _emu_case('h2o', emu_lib)
    dm = _inputs(nao)['general0'][0]
    wj, wk = d0.get_jk(dm, hermi=0)
    vj = np.zeros_like(wj)
    vk = np.zeros_like(wk)
    for rank in range(2):
        d = DF(mol, aux, libpath=emu_lib, shard=(rank, 2)).set_device_rows(5).build()
        n_dev, n_host = d.row_split()
        assert n_dev == 5 and n_host > 0
        _set_kblock(d, 4)
        pj, pk = d.get_jk(dm, hermi=0)
        vj += pj
        vk += pk
    assert abs(vj - wj).max() < 1e-12 and abs(vk - wk).max() < 1e-12


def test_device_rows_argument_checked(emu_lib):
    mol, aux, ref, nao, d0 = _emu_case('h2o', emu_lib)
    h = d0._handle
    assert h.lib.b200jk_df_set_device_rows(h._h, -2) != 0


# ---- GPU -------------------------------------------------------------------------------------------------------------------

def _gpu_c60(cap):
    import df_size_check as S
    z = S.load('c60')
    mol = gto.M(atom=geometry('c60'), basis='def2-svp')
    return S, z, mol, DF(mol).set_device_rows(cap).build()


def _check_size_fixture(S, z, d, mol, engines=('tcgen05', 'dgemm')):
    """Columns and J/K of the fixture within 1e-9 (orbital-tagged and general density, per K engine), and the two K
    algorithms against each other on the SCF-like density."""
    dc = S.check_columns(d, z)
    assert dc < 1e-9, ('cderi columns', dc)
    c = S.slab_coeff(z)
    occ = np.full(c.shape[1], 2.0)
    dm = 2.0 * c.dot(c.T)
    out = {}
    for eng in engines:
        d.set_k_engine(eng, 7)
        vj1, vk1 = d.get_jk(TaggedDM(dm, mo_coeff=c, mo_occ=occ), hermi=1)
        r1 = S.compare_jk(z, vj1, vk1)
        assert max(r1['max_abs_dJ'], r1['max_abs_dK'], r1['max_abs_dK_diag']) < 1e-9, (eng, 'orbital-tagged', r1)
        vj2, vk2 = d.get_jk(dm, hermi=1)
        r2 = S.compare_jk(z, vj2, vk2)
        assert max(r2['max_abs_dJ'], r2['max_abs_dK'], r2['max_abs_dK_diag']) < 1e-9, (eng, 'general density', r2)
        out[eng] = (vj1, vk1, vj2, vk2)
    d.set_k_engine('tcgen05', 7)
    rng = np.random.RandomState(1)
    co, _ = np.linalg.qr(rng.standard_normal((mol.nao, int(z['nocc']))))
    dms = 2.0 * co.dot(co.T)
    _, vk3 = d.get_jk(TaggedDM(dms, mo_coeff=co, mo_occ=np.full(co.shape[1], 2.0)), hermi=1, with_j=False)
    _, vk4 = d.get_jk(dms, hermi=1, with_j=False)
    assert abs(vk3 - vk4).max() < 1e-9, abs(vk3 - vk4).max()
    return out, dc


_C60_RESIDENT = {}


def _c60_resident():
    if not _C60_RESIDENT:
        S, z, mol, d = _gpu_c60(-1)
        try:
            assert d.row_split()[1] == 0
            _C60_RESIDENT['naux'] = d.get_naoaux()
            _C60_RESIDENT['out'] = _check_size_fixture(S, z, d, mol)[0]
        finally:
            d.reset()
    return _C60_RESIDENT['out']


@pytest.mark.gpu
@pytest.mark.parametrize('frac', ['all_host', 'half_host'])
def test_c60_forced_split_gpu(frac):
    """C60/def2-SVP with no / half of the rows on the device: fixture columns and J/K within 1e-9 for both K engines, and J/K
    within 1e-10 of the all-resident build (only the K-range partition and the summation order differ)."""
    want = _c60_resident()
    naux = _C60_RESIDENT['naux']
    S, z, mol, d = _gpu_c60(0 if frac == 'all_host' else naux // 2)
    try:
        cap = 0 if frac == 'all_host' else naux // 2
        assert d.row_split() == (cap, naux - cap)
        got, dc = _check_size_fixture(S, z, d, mol)
        for eng in got:
            for a, b in zip(got[eng], want[eng]):
                assert abs(a - b).max() < 1e-10, (eng, abs(a - b).max())
        st = d.stream_stats()
        npair = mol.nao * (mol.nao + 1) // 2
        assert st['bytes'] == (naux - cap) * npair * 8 and st['copy_ms'] > 0, st
        print('c60 %s: cols %.1e, stream %s' % (frac, dc, st))
    finally:
        d.reset()


def _c60_split_blocked():
    """Half of the C60 rows on the host with K blocks of 64 rows (several staged blocks per call) and resident slices capped."""
    want = _c60_resident()
    S, z, mol, d = _gpu_c60(_C60_RESIDENT['naux'] // 2)
    try:
        h = d._handle
        h.check(h.lib.b200jk_df_set_kblock(h._h, 64, 300), 'b200jk_df_set_kblock')
        got, _ = _check_size_fixture(S, z, d, mol)
        for eng in got:
            for a, b in zip(got[eng], want[eng]):
                assert abs(a - b).max() < 1e-10, (eng, abs(a - b).max())
    finally:
        d.reset()


@pytest.mark.gpu
def test_c60_split_kblock_gpu():
    _c60_split_blocked()


@pytest.mark.gpu
def test_c60_split_unfused_y_gpu():
    """The blocked split with B200JK_NO_YFUSE=1, in a fresh process because the variable is read once per process."""
    here = os.path.dirname(os.path.abspath(__file__))
    code = 'import sys; sys.path[:0] = [%r, %r]; import test_df_outcore as T; T._c60_split_blocked()' % (here, os.path.dirname(here))
    r = subprocess.run([sys.executable, '-c', code], env=dict(os.environ, B200JK_NO_YFUSE='1'), capture_output=True, text=True,
                       timeout=1800)
    assert r.returncode == 0, r.stdout[-2000:] + r.stderr[-4000:]


@pytest.mark.gpu
@pytest.mark.parametrize('name,geom,basis', [('c60', 'c60', 'def2-svp'), ('taxol_svp', 'taxol', 'def2-svp')])
def test_fitting_tensor_stays_on_device_gpu(name, geom, basis):
    """The automatic split leaves a tensor that fits entirely in HBM: nothing is streamed."""
    d = DF(gto.M(atom=geometry(geom), basis=basis)).build()
    try:
        assert d.row_split()[1] == 0, d.row_split()
    finally:
        d.reset()


def _mem_available():
    with open('/proc/meminfo') as f:
        for line in f:
            if line.startswith('MemAvailable:'):
                return int(line.split()[1]) * 1024
    return 0


@pytest.mark.gpu
def test_taxol_tzvp_one_gpu():
    """Taxol/def2-TZVP (111 GB tensor) on one 80 GB GPU with the automatic split, against the size fixture."""
    import torch
    import df_size_check as S
    z = S.load('taxol')
    mol = gto.M(atom=geometry('taxol'), basis='def2-tzvp')
    naux, nao = int(z['naux']), mol.nao
    tensor = naux * nao * (nao + 1) // 2 * 8
    total = torch.cuda.get_device_properties(0).total_memory
    host_needed = tensor - 0.8 * total        # at least the part beyond the device's memory
    if _mem_available() < host_needed:
        print('skipped: MemAvailable %.1f GB is below the %.1f GB of pinned rows needed' % (_mem_available() / 1e9, host_needed / 1e9))
        pytest.skip('MemAvailable %.1f GB below the %.1f GB of pinned host rows needed' % (_mem_available() / 1e9, host_needed / 1e9))
    d = DF(mol).build()
    try:
        n_dev, n_host = d.row_split()
        assert n_host > 0 and n_dev + n_host == naux, (n_dev, n_host)
        out, dc = _check_size_fixture(S, z, d, mol, engines=('tcgen05',))
        print('taxol/def2-tzvp split %s, cols %.1e, stream %s' % ((n_dev, n_host), dc, d.stream_stats()))
    finally:
        d.reset()
