"""The int8-slice DF-K engine on the GPU, kernel by kernel (b200jk_i8engine_test) against the bit-exact numpy model of
tests/i8model.py and the exact product, and the DF-level K build with forced blocking (b200jk_df_set_kblock)."""
import ctypes
import os
import subprocess
import sys

import numpy as np
import pytest

import i8model as M

H2O = 'O 0 0 0; H 0 -0.757 0.587; H 0 0.757 0.587'


@pytest.fixture(scope='module')
def handle():
    from pyscf_b200 import gto, lib
    mol = gto.M(atom=H2O, basis='sto-3g')
    h = lib.Handle(mol._atm, mol._bas, np.array(mol._env, dtype=np.float64))
    yield h
    h.close()


def run(h, stage, ns, a, k, packed=False, b=None, a_rowmax=None, a_row0=0, m=0, inner=0, y_ncolp=0, symmetric=0, kb_per=0):
    """b200jk_i8engine_test with every output requested; returns a dict of numpy arrays."""
    from pyscf_b200 import lib
    a = np.ascontiguousarray(a, dtype=np.float64)
    ra = a.shape[0]
    rows_a = ra * k if packed else ra
    Rpa, Kp = M.stack_rows(rows_a), M.pad_to(k, M.BK)
    out = {'qa': np.zeros((ns, Rpa, Kp), np.int8), 'ea': np.zeros(Rpa, np.int32)}
    t = lib.I8Test(stage=stage, packed=int(packed), ns=ns, a=lib.dptr(a), ra=ra, k=k, a_row0=a_row0, m=m, inner=inner,
                   y_ncolp=y_ncolp, symmetric=symmetric, kb_per=kb_per)
    if a_rowmax is not None:
        a_rowmax = np.ascontiguousarray(a_rowmax, dtype=np.float64)
        t.a_rowmax = lib.dptr(a_rowmax)
    if packed:
        out['rowexp'] = np.zeros((ra, k), np.int32)
        out['rownorm2'] = np.zeros((ra, k), np.float32)
        t.rowexp = lib.iptr(out['rowexp'])
        t.rownorm2 = out['rownorm2'].ctypes.data_as(ctypes.POINTER(ctypes.c_float))
    if b is not None:
        b = np.ascontiguousarray(b, dtype=np.float64)
        t.b, t.rb = lib.dptr(b), b.shape[0]
        Rpb = M.stack_rows(b.shape[0])
        out['qb'], out['eb'] = np.zeros((ns, Rpb, Kp), np.int8), np.zeros(Rpb, np.int32)
        t.qb, t.eb = out['qb'].ctypes.data, lib.iptr(out['eb'])
        if stage == 1 and y_ncolp:
            Rpy, Kpy = M.stack_rows(inner), M.pad_to(m // inner * y_ncolp, M.BK)
            out['qy'], out['ey'] = np.zeros((ns, Rpy, Kpy), np.int8), np.zeros(Rpy, np.int32)
            t.qy, t.ey = out['qy'].ctypes.data, lib.iptr(out['ey'])
        elif stage == 1:
            rows = inner if inner > 0 else m
            ldc = (m + inner - 1) // inner * b.shape[0] if inner > 0 else b.shape[0]
            out['c'], out['rowmax'] = np.zeros((rows, ldc)), np.zeros(rows)
            t.c, t.rowmax = lib.dptr(out['c']), lib.dptr(out['rowmax'])
        else:
            out['c'] = np.zeros((ra, b.shape[0]))
            t.c = lib.dptr(out['c'])
    t.qa, t.ea = out['qa'].ctypes.data, lib.iptr(out['ea'])
    h.check(h.lib.b200jk_i8engine_test(h._h, ctypes.byref(t)), 'b200jk_i8engine_test')
    return out


def same_stack(out_q, out_e, S):
    assert out_q.shape == S.q.shape and out_e.shape == S.E.shape
    assert (out_e == S.E).all()
    bad = np.argwhere(out_q != S.q)
    assert bad.size == 0, ('digits differ', bad[:5], out_q[tuple(bad[0])], S.q[tuple(bad[0])])


def edge_rows(rng, K):
    """Rows at the edges of the slicing: top digit 64, .5 ties, powers of two, a zero row, one non-zero, 2^+-300 spans,
    a subnormal row maximum, rows near the top of the range."""
    r = [np.full(K, 1.0 - 2.0 ** -53), np.full(K, 0.75 + 2.0 ** -8), np.ldexp(1.0, rng.randint(-40, 40, K)) * rng.choice([-1, 1], K),
         np.zeros(K), np.eye(1, K, K // 2)[0] * -3.0, rng.standard_normal(K) * np.ldexp(1.0, rng.randint(-300, 300, K)),
         rng.standard_normal(K) * 2.0 ** -1070, rng.standard_normal(K) * 2.0 ** 1020, rng.standard_normal(K) * 2.0 ** -1000]
    return np.array(r)


# ------------------------------------------------------------------------------------------------- slicing kernels
@pytest.mark.gpu
@pytest.mark.parametrize('ns', range(1, 9))
@pytest.mark.parametrize('R,K', [(37, 200), (9, 8192 + 5), (300, 129)])
def test_split_rows_bit_exact(handle, ns, R, K):
    """split_rows (one warp per row; the long-row kernels for K >= 8192 with fewer than 4096 rows): digits, exponents and
    zero pads equal the model."""
    rng = np.random.RandomState(R + ns)
    X = rng.standard_normal((R, K)) * np.exp(rng.uniform(-20, 20, (R, 1)))
    X[:9] = edge_rows(rng, K)
    out = run(handle, 0, ns, X, K)
    same_stack(out['qa'], out['ea'], M.slice_rows(X, ns))


@pytest.mark.gpu
@pytest.mark.parametrize('ns', [3, 7, 8])
def test_split_rows_premax_bit_exact(handle, ns):
    """split_rows_premax with row maxima given by the producer (exact maxima, and larger ones: a looser exponent)."""
    rng = np.random.RandomState(ns)
    X = rng.standard_normal((20, 8200))
    X[:9] = edge_rows(rng, 8200)
    mx = np.abs(X).max(axis=1)
    mx[10:] *= 3.0
    out = run(handle, 0, ns, X, 8200, a_rowmax=mx)
    same_stack(out['qa'], out['ea'], M.slice_rows(X, ns, rowmax=mx))


def packed_tensor(rng, nr, nao):
    """Packed rows cderi[P][a(a+1)/2+b] with rows at the exponent edges: tiny (2^-1000: the scale 2^(48-e) leaves the range
    of pow2i), subnormal, and an all-zero auxiliary row."""
    npair = nao * (nao + 1) // 2
    c = rng.standard_normal((nr, npair)) * np.exp(rng.uniform(-5, 5, (nr, 1)))
    c[0] *= 2.0 ** -1000
    c[1] *= 2.0 ** -1065
    c[2] = 0.0
    c[3, ::7] = 0.75 + 2.0 ** -8
    return c


@pytest.mark.gpu
@pytest.mark.parametrize('ns', range(1, 9))
@pytest.mark.parametrize('nao', [24, 70, 130])
def test_split_packed_bit_exact(handle, ns, nao):
    """packed_rowexp + split_packed (NS7 mantissa path at ns = 7, generic mantissa path below, rint digits at ns = 8) with
    nao not a multiple of 64 / 128: row exponents, digits and zero pads equal the model."""
    rng = np.random.RandomState(nao + ns)
    c = packed_tensor(rng, 6, nao)
    out = run(handle, 0, ns, c, nao, packed=True)
    S, rowexp = M.slice_packed(c, nao, ns)
    EXP_NONE = np.int32(-0x7f7f7f80)                                    # memset 0x80: the row has no non-zero
    assert (out['rowexp'][2] == EXP_NONE).all()
    assert (np.where(out['rowexp'] == EXP_NONE, 0, out['rowexp']) == rowexp).all()
    same_stack(out['qa'], out['ea'], S)
    X = M.unpack_rows(c, nao)
    n2 = (X.astype(np.float64) ** 2).astype(np.float32).sum(axis=1)
    assert np.allclose(out['rownorm2'].reshape(-1), n2, rtol=1e-5, atol=0)


# ------------------------------------------------------------------------------------------------- GEMM, one K range
SIZES = [1, 31, 32, 33, 127, 128, 129, 255, 256, 257]
KS = [1, 127, 128, 129, 2047, 2048, 8191, 8192 + 5]
GRID = [(SIZES[i], SIZES[(3 * i + j) % 10], KS[j], 1 + (i + 2 * j) % 8) for i in range(10) for j in range(0, 8, 2)] + \
       [(SIZES[(i + 5) % 10], SIZES[i], KS[j], 1 + (i + j) % 8) for i in range(10) for j in range(1, 8, 2)]


@pytest.mark.gpu
@pytest.mark.parametrize('Mr,N,K,ns', GRID)
def test_gemm_one_range_bit_exact(handle, Mr, N, K, ns):
    """Stage 2 (accumulate from zero, K forced into one range) and stage 1 (plain stores) equal the model bit for bit over
    partial tiles, K around the 128-byte blocks and the long-row slicing."""
    rng = np.random.RandomState(Mr * 1000 + N + K)
    A = rng.standard_normal((Mr, K)) * np.exp(rng.uniform(-8, 8, (Mr, 1)))
    B = rng.standard_normal((N, K)) * np.exp(rng.uniform(-8, 8, (N, 1)))
    Sa, Sb = M.slice_rows(A, ns), M.slice_rows(B, ns)
    out = run(handle, 2, ns, A, K, b=B, kb_per=Sa.Kp // M.BK)
    C, _ = M.stage2(Sa, Sb)
    assert (out['c'] == C).all(), np.abs(out['c'] - C).max()
    out1 = run(handle, 1, ns, A, K, b=B, m=Mr)
    assert (out1['c'] == C).all()
    assert (out1['rowmax'] == np.abs(C).max(axis=1)).all()


@pytest.mark.gpu
@pytest.mark.parametrize('ns', [2, 7, 8])
def test_gemm_stage1_scatter_row_block(handle, ns):
    """Stage 1 on a row block of the stack (a_row0 != 0) with the transposed scatter and the row maxima, as DF-K's plain
    stage 1 uses them (B200JK_NO_YFUSE)."""
    inner, N, K = 45, 37, 300
    rng = np.random.RandomState(ns)
    A = rng.standard_normal((5 * inner, K)) * np.exp(rng.uniform(-4, 4, (5 * inner, 1)))
    B = rng.standard_normal((N, K))
    Sa, Sb = M.slice_rows(A, ns), M.slice_rows(B, ns)
    out = run(handle, 1, ns, A, K, b=B, a_row0=inner, m=3 * inner, inner=inner)
    C, rowmax = M.stage1(Sa, Sb, a_row0=inner, m=3 * inner, inner=inner)
    assert (out['c'] == C).all() and (out['rowmax'] == rowmax).all()


@pytest.mark.gpu
@pytest.mark.parametrize('n,K,ns,same', [(257, 300, 7, True), (257, 300, 7, False), (129, 2100, 5, False), (33, 129, 8, True)])
def test_gemm_symmetric_bit_exact(handle, n, K, ns, same):
    """Symmetric mode (only tiles touching the upper triangle, only n >= m written) with B = A and with B != A (hermi = 1
    general densities)."""
    rng = np.random.RandomState(n + K)
    A = rng.standard_normal((n, K))
    B = A.copy() if same else rng.standard_normal((n, K))
    Sa, Sb = M.slice_rows(A, ns), M.slice_rows(B, ns)
    out = run(handle, 2, ns, A, K, b=B, symmetric=1, kb_per=Sa.Kp // M.BK)
    C, _ = M.stage2(Sa, Sb, symmetric=True)
    assert (out['c'] == C).all()


# ------------------------------------------------------------------------------------------------- several K ranges
@pytest.mark.gpu
@pytest.mark.parametrize('kb_per,sym', [(1, 0), (3, 0), (2, 1), (0, 0)])
def test_gemm_k_ranges(handle, kb_per, sym):
    """K ranges (forced, and the automatic choice for a long K) meet in fp64 atomics: within the re-association bound of
    the model's per-range values."""
    rng = np.random.RandomState(kb_per)
    n, K, ns = 150, 40 * 128 + 17, 7
    A = rng.standard_normal((n, K))
    B = A + 0.1 * rng.standard_normal((n, K)) if sym else rng.standard_normal((n - 20, K))
    Sa, Sb = M.slice_rows(A, ns), M.slice_rows(B, ns)
    out = run(handle, 2, ns, A, K, b=B, symmetric=sym, kb_per=kb_per)
    if kb_per:
        C, parts = M.stage2(Sa, Sb, symmetric=bool(sym), kb_per=kb_per)
        tol = M.ranges_bound(parts)                 # every range is bit-exact; only the order of the fp64 atomics is free
    else:                                           # automatic ranges: any partition is within a few roundings of one range
        C, _ = M.stage2(Sa, Sb, symmetric=bool(sym))
        tol = 2.0 ** -46 * np.abs(A) @ np.abs(B).T
    assert (np.abs(out['c'] - C) <= tol).all()


# ------------------------------------------------------------------------------------------------- fused Y
@pytest.mark.gpu
@pytest.mark.parametrize('ns', [5, 6, 7, 8])
@pytest.mark.parametrize('nao,ncol', [(24, 5), (70, 33), (130, 16)])
def test_stage1_fused_y(handle, ns, nao, ncol):
    """The Y slices cut in the stage-1 epilogue equal the model given the kernel's own exponent bounds Ey; Ey is a true
    bound of the exact Y and no looser than the documented Cauchy-Schwarz margin (factor 1.001 on float32 norms)."""
    rng = np.random.RandomState(nao + ns)
    nr = 7
    c = rng.standard_normal((nr, nao * (nao + 1) // 2)) * np.exp(rng.uniform(-3, 3, (nr, 1)))
    right = rng.standard_normal((ncol, nao))
    ncolp = M.pad_to(ncol, 16)
    r0 = 2                                                              # block = packed rows 2 .. 6
    out = run(handle, 1, ns, c, nao, packed=True, b=right, a_row0=r0 * nao, m=(nr - r0) * nao, inner=nao, y_ncolp=ncolp)
    SA, _ = M.slice_packed(c, nao, ns)
    SC = M.slice_rows(right, ns)
    same_stack(out['qa'], out['ea'], SA)
    Ey = out['ey'][:nao].astype(np.int64)
    SY = M.stage1_y(SA, SC, Ey, r0 * nao, (nr - r0) * nao, nao, ncolp)
    same_stack(out['qy'], out['ey'], SY)
    X = M.unpack_rows(c, nao).reshape(nr, nao, nao)[r0:]
    Y = np.einsum('pab,ib->api', X, right)                              # [nao][P][i]
    ymax = np.abs(Y).reshape(nao, -1).max(axis=1)
    assert (ymax < np.ldexp(1.0, Ey.astype(np.int32))).all()
    cs = np.sqrt((X ** 2).sum(axis=2).max(axis=0) * (right ** 2).sum(axis=1).max())
    assert (np.ldexp(1.0, (Ey - 1).astype(np.int32)) <= 1.0012 * cs).all()


# ------------------------------------------------------------------------------------------------- exact products, defects
@pytest.mark.gpu
@pytest.mark.parametrize('ns', [4, 7, 8])
def test_engine_against_exact(handle, ns):
    """The whole engine (slicing + stage 2) against the exact product of the fp64 inputs, within the model's bound, on
    structured rows including exponents far outside the range of a single 2^e multiplier."""
    rng = np.random.RandomState(ns)
    K = 60
    A = np.vstack([edge_rows(rng, K), rng.standard_normal((12, K)) * np.exp(rng.uniform(-30, 30, (12, 1)))])
    B = np.vstack([rng.standard_normal((10, K)) * 2.0 ** -540, edge_rows(rng, K)[[0, 1, 2, 4, 5, 8]], rng.standard_normal((4, K))])
    out = run(handle, 2, ns, A, K, b=B)
    Sa, Sb = M.slice_rows(A, ns), M.slice_rows(B, ns)
    C, _ = M.stage2(Sa, Sb)
    ref = M.exact_abt(A, B)
    fin = np.isfinite(ref)
    assert (out['c'][~fin] == ref[~fin]).all()
    assert (out['c'] == C).all()
    err = np.abs(np.where(fin, out['c'], 0) - np.where(fin, ref, 0))
    assert (err <= M.product_bound(ns, K, Sa.E[:Sa.R], Sb.E[:Sb.R])).all()


@pytest.mark.gpu
def test_tiny_and_huge_rows(handle):
    """Row exponents whose sum leaves [-1022, 1023]: products underflow to subnormals / 0 and overflow to inf like the exact
    product, in the plain, the accumulate and the fused-Y epilogue and in split_rows for a subnormal row maximum."""
    rng = np.random.RandomState(5)
    K = 40
    A = np.vstack([rng.standard_normal(K) * 2.0 ** s for s in (-540, -530, -1060, 500, 0)])
    B = np.vstack([rng.standard_normal(K) * 2.0 ** s for s in (-540, -520, 0, 540)])
    ref = M.exact_abt(A, B)
    for stage in (1, 2):
        out = run(handle, stage, 7, A, K, b=B, m=A.shape[0])
        fin = np.isfinite(ref)
        assert (out['c'][~fin] == ref[~fin]).all()
        Sa, Sb = M.slice_rows(A, 7), M.slice_rows(B, 7)
        assert (np.abs(out['c'] - ref)[fin] <= M.product_bound(7, K, Sa.E[:5], Sb.E[:4])[fin]).all()


@pytest.mark.gpu
def test_int32_bound_enforced(handle):
    """Digits all 64 (ns = 1) over K = 2^19: one group sum would be exactly 2^31.  Stage 2 splits K so that every range is
    exact; a forced single range and stage 1 (always one range) are refused instead of wrapping."""
    K = 1 << 19
    A = np.full((1, K), 1.0 - 2.0 ** -10)
    out = run(handle, 2, 1, A, K, b=A)
    assert out['c'][0, 0] == float(K) * (64 * 64) * 2.0 ** -12            # exact: 2^31 2^-12
    with pytest.raises(RuntimeError, match='int32'):
        run(handle, 2, 1, A, K, b=A, kb_per=K // 128)
    with pytest.raises(RuntimeError, match='int32'):
        run(handle, 1, 1, A, K, b=A, m=1)


# ------------------------------------------------------------------------------------------------- DF level
def _df_setup(name):
    from pyscf_b200 import gto
    from pyscf_b200.df import DF
    from pyscf_b200.gto.mole import geometry, make_auxmol
    from oracle import oracle as O
    if name == 'h2o':
        mol, aux = gto.M(atom=H2O, basis='cc-pvdz'), 'weigend'
    else:
        mol, aux = gto.M(atom=geometry('benzene'), basis='def2-svp'), 'def2-svp-jkfit'
    d = DF(mol, aux).build()
    ref, nao = O.cholesky_eri(mol, make_auxmol(mol, aux))
    return d, ref, nao, O


def _df_checks(name, cases):
    """K of the int8 engine under forced blocking == oracle within the model-derived bound.  The blocking changes the
    exponent bounds of Y (maxima over the block's auxiliary rows), hence the slicing: forced and automatic blocking agree
    within the sum of their bounds, and to 1e-12 at 8 slices.  cases: (ns, kblock, resident)."""
    from pyscf_b200.df import TaggedDM
    from test_i8model import model_df_k
    d, ref, nao, O = _df_setup(name)
    h = d._handle
    rng = np.random.RandomState(1)
    c1, c2 = (np.linalg.qr(rng.standard_normal((nao, 6)))[0] * np.sqrt(2.0) for _ in range(2))
    dm_g = rng.random_sample((2, nao, nao))
    dm_s = dm_g + dm_g.transpose(0, 2, 1)
    dms_t = np.array([c1 @ c1.T, c2 @ c2.T])
    inputs = {'tagged': (TaggedDM(dms_t, mo_coeff=np.array([c1, c2]), mo_occ=np.full((2, 6), 1.0)), 1, dms_t),
              'general0': (dm_g, 0, dm_g), 'general1': (dm_s, 1, dm_s)}
    naux = d.get_naoaux()
    for ns in sorted({c[0] for c in cases}):
        d.set_k_engine('tcgen05', ns)
        h.check(h.lib.b200jk_df_set_kblock(h._h, -1, -1), 'b200jk_df_set_kblock')
        auto = {k: d.get_jk(v[0], hermi=v[1], with_j=False)[1] for k, v in inputs.items()}
        tol = {}
        for kind, (_, hermi, dms) in inputs.items():
            for s in range(2):
                occ = [c1, c2][s] if kind == 'tagged' else None
                Km, Kb = model_df_k(ref, nao, dms[s], ns, occ=occ, hermi=hermi)
                tol[kind, s] = Kb + 1e-13 * np.abs(Km).max()
        for _, kbl, res in [c for c in cases if c[0] == ns]:
            res = min(res, naux) if res >= 0 else res
            h.check(h.lib.b200jk_df_set_kblock(h._h, kbl, res), 'b200jk_df_set_kblock')
            for kind, (dm, hermi, dms) in inputs.items():
                vk = d.get_jk(dm, hermi=hermi, with_j=False)[1]
                for s in range(2):
                    rk = O.df_get_jk(ref, nao, dms[s])[1]
                    assert (np.abs(vk[s] - rk) <= tol[kind, s]).all(), (name, ns, kbl, res, kind, s)
                for s in range(2):
                    assert (np.abs(vk[s] - auto[kind][s]) <= 2 * tol[kind, s]).all(), (name, ns, kbl, res, kind, s)
                if ns == 8:
                    assert np.abs(vk - auto[kind]).max() < 1e-12, (name, ns, kbl, res, kind)
                if ns == 7:
                    assert np.abs(vk - np.array([O.df_get_jk(ref, nao, x)[1] for x in dms])).max() < 1e-9
    h.check(h.lib.b200jk_df_set_kblock(h._h, -1, -1), 'b200jk_df_set_kblock')


DF_CASES = {'h2o': [(7, 1, -1), (7, 3, 0), (7, 7, 10), (7, 3, 13), (5, 3, 10), (6, 7, 0), (8, 1, 5), (8, 7, -1)],
            'benzene': [(7, 1, -1), (7, 3, 0), (7, 7, 10), (7, 3, 13), (8, 7, 5)]}     # the model of 5, 6 slices costs minutes here


@pytest.mark.gpu
@pytest.mark.parametrize('name', ['h2o', 'benzene'])
def test_df_k_blocking(name):
    """Several K blocks (1, 3, 7 auxiliary rows: partial last blocks, the right factor reused across blocks for one density
    per orbital set), all / no / some rows resident (boundaries inside a block), n_dm = 2, tagged and general densities,
    hermi 0 and 1, 5 to 8 slices."""
    _df_checks(name, DF_CASES[name])


@pytest.mark.gpu
def test_df_k_unfused_y():
    """The same DF checks with B200JK_NO_YFUSE=1 (fp64 Y, its slices cut by split_rows / split_rows_premax after stage 1),
    in a fresh process because the variable is read once per process."""
    here = os.path.dirname(os.path.abspath(__file__))
    code = ('import sys; sys.path[:0] = [%r, %r]; import test_i8gemm as T; '
            'T._df_checks("h2o", [(7, 3, 0), (7, 7, 13), (6, 1, -1)]); T._df_checks("benzene", [(7, 7, 10)])'
            % (here, os.path.dirname(here)))
    env = dict(os.environ, B200JK_NO_YFUSE='1')
    r = subprocess.run([sys.executable, '-c', code], env=env, capture_output=True, text=True, timeout=900)
    assert r.returncode == 0, r.stdout[-2000:] + r.stderr[-4000:]
