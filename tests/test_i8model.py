"""CPU tests of the int8-slice DF-K engine's arithmetic (tests/i8model.py): the model against exact products, the int32 bound
of the slice-pair sums, and the DF-K algorithm of the engine against the oracle's FP64 algebra."""
from fractions import Fraction

import numpy as np
import pytest

import i8model as M


def structured_rows(rng, K):
    """Rows where slicing goes wrong: .5 ties at every digit, values rounding up to a top digit of 64, exact powers of two,
    a zero row, single non-zeros, rows spanning 2^-300 .. 2^300, subnormals and values near the top of the range."""
    rows = []
    rows.append(np.full(K, 1.0 - 2.0 ** -53))                           # rounds up to a top digit of 64
    r = np.zeros(K); r[:] = 0.75 + 2.0 ** -8                            # a .5 tie below the top digit
    rows.append(r)
    rows.append(np.ldexp(1.0, rng.randint(-40, 40, K)) * rng.choice([-1, 1], K))     # powers of two
    rows.append(np.zeros(K))
    r = np.zeros(K); r[K // 2] = -3.0; rows.append(r)                   # a single non-zero
    rows.append(rng.standard_normal(K) * np.ldexp(1.0, rng.randint(-300, 300, K)))    # spans 2^+-300
    rows.append(rng.standard_normal(K) * 2.0 ** -1070)                  # subnormal row maximum
    rows.append(rng.standard_normal(K) * 2.0 ** 1020)                   # near the top of the range
    t = np.zeros(K)                                                      # ties at every digit position
    for s in range(8):
        t += 2.0 ** (-7 * s - 1)
    rows.append(t * 0.5)
    rows.append(rng.standard_normal(K))
    return np.array(rows)


@pytest.mark.parametrize('ns', range(1, 9))
@pytest.mark.parametrize('convention', ['rint', 'mantissa', 'yfused'])
def test_digits_represent_rows(ns, convention):
    """Every row is represented to half a unit of its last digit: |x - value(digits)| <= 2^(e - 7 ns), i.e. 2^-48 of the row
    maximum for ns = 7 (DESIGN.md §4.4); top digits are within +-64, lower ones within the convention's range."""
    rng = np.random.RandomState(ns)
    X = structured_rows(rng, 37)
    if convention == 'mantissa' and ns == 8:
        pytest.skip('split_packed uses rint digits for ns = 8')
    if convention == 'rint':
        E = M.row_exponents(X)
        q = M.digits_rint(X, E, ns)
    elif convention == 'mantissa':
        E = M.row_exponents(X)
        q = M.digits_mantissa(X, E, ns)
    else:
        E = M.row_exponents(X)
        q = M.digits_yfused(np.ldexp(X, (6 - E)[:, None].astype(np.int32)), ns)
    assert np.abs(q[0].astype(int)).max() <= 64
    lo = q[1:].astype(int)
    if convention == 'mantissa':
        assert lo.min(initial=0) >= 0 and lo.max(initial=0) <= 127
    else:
        assert np.abs(lo).max(initial=0) <= 64
    for i in range(X.shape[0]):
        for j in range(X.shape[1]):
            x = Fraction(float(X[i, j]))
            v = sum(Fraction(int(q[s, i, j])) * Fraction(2) ** (int(E[i]) - 6 - 7 * s) for s in range(ns))
            assert abs(v - x) <= Fraction(2) ** (int(E[i]) - 7 * ns), (convention, ns, i, j)


def test_row_exponents_are_bounds():
    rng = np.random.RandomState(0)
    X = structured_rows(rng, 20)
    E = M.row_exponents(X)
    for i in range(X.shape[0]):
        mx = np.abs(X[i]).max()
        if mx > 0:
            assert mx < 2.0 ** int(E[i]) if E[i] < 1024 else True
            assert mx >= np.ldexp(1.0, int(E[i]) - 1)
        else:
            assert E[i] == 0
    # packed exponents: frexp exponent for normal numbers, -1022 (a bound, not the exponent) for subnormals
    assert M.frexp_exp(np.array([1.0, 0.75, 2.0 ** -1074, 3.0 * 2 ** 1000])).tolist() == [1, 0, -1022, 1002]


@pytest.mark.parametrize('ns', [1, 2, 4, 6, 7, 8])
@pytest.mark.parametrize('packed', [False, True])
def test_model_against_exact_product(ns, packed):
    """The model's C = A B^T is within its stated bound (product_bound) of the exact product, on random and structured
    operands; the bound is not vacuous (the observed error uses at least 1/2^12 of it somewhere)."""
    rng = np.random.RandomState(10 * ns + packed)
    K = 45
    A = np.vstack([structured_rows(rng, K), rng.standard_normal((6, K)) * np.exp(rng.uniform(-30, 30, (6, 1)))])
    B = np.vstack([rng.standard_normal((9, K)) * np.exp(rng.uniform(-20, 20, (9, 1))), structured_rows(rng, K)[[0, 1, 2, 4, 8, 9]]])
    Sa = M.slice_rows(A, ns)
    if packed and ns <= 7:       # the mantissa digits of split_packed on the same rows
        Sa = M.Stack(M.digits_mantissa(A, M.row_exponents(A), ns), M.row_exponents(A), dmax=127)
    Sb = M.slice_rows(B, ns)
    _, C = M.product(Sa, Sb)
    ref = M.exact_abt(A, B)
    bound = M.product_bound(ns, K, Sa.E[:Sa.R], Sb.E[:Sb.R], Sa.dmax, Sb.dmax)
    finite = np.isfinite(ref)
    assert (C[~finite] == ref[~finite]).all()
    err = np.where(finite, np.abs(np.where(finite, C, 0.0) - np.where(finite, ref, 0.0)), 0.0)
    assert (err <= bound).all(), (err / bound).max()
    assert (err / bound).max() > 2.0 ** -12


def test_extreme_exponents():
    """Products that underflow to subnormals or 0 and products of huge rows: the model (ldexp scaling, one rounding) equals
    the exact product to its bound, no wrapped 2^e values (the kernel's defect before scale2 / pow2_split)."""
    K = 16
    rng = np.random.RandomState(3)
    A = np.vstack([rng.standard_normal(K) * 2.0 ** -540, rng.standard_normal(K) * 2.0 ** -1060, rng.standard_normal(K) * 2.0 ** 500])
    B = np.vstack([rng.standard_normal(K) * 2.0 ** -540, rng.standard_normal(K) * 2.0 ** -20, rng.standard_normal(K) * 2.0 ** 540])
    for ns in (5, 7, 8):
        Sa, Sb = M.slice_rows(A, ns), M.slice_rows(B, ns)
        _, C = M.product(Sa, Sb)
        ref = M.exact_abt(A, B)
        bound = M.product_bound(ns, K, Sa.E[:3], Sb.E[:3])
        ok = np.isfinite(ref)
        assert (np.abs(C - ref)[ok] <= bound[ok]).all()
        assert np.isinf(C[2, 2]) and np.isinf(ref[2, 2])            # overflows like the exact product
        assert C[0, 0] == 0.0 or abs(C[0, 0]) < 2.0 ** -1000        # underflows, never a large wrong value


def test_int32_bound():
    """Operands whose digits are all +-64 (top digit of 64 on every slice) reach the int32 limit exactly where the bound
    ns k dmax_a dmax_b <= 2^31 - 1 says: at df.cu's old stage-2 block size 2^19 / ns the group sum is 2^31, one past int32."""
    for ns in (1, 2, 7):
        k_old = (1 << 19) // ns
        assert not M.int32_ok(ns, k_old, 64, 64) or ns * k_old * 4096 < 2 ** 31
        k_new = ((1 << 31) - 1) // (4096 * ns)
        assert M.int32_ok(ns, k_new, 64, 64)
    # ns = 1 at K = 2^19: one slice pair, every digit 64 -> 64 * 64 * 2^19 = 2^31
    ns, K = 1, 1 << 19
    X = np.full((1, K), 1.0 - 2.0 ** -10)
    S = M.slice_rows(X, ns)
    assert (S.q[0, 0, :K] == 64).all()
    with pytest.raises(OverflowError):
        M.group_sums(S.q[:, :1], S.q[:, :1])
    assert M.group_sums(S.q[:, :1], S.q[:, :1], wrap=True)[0, 0, 0] == -2 ** 31      # what the kernel would have returned
    assert M.group_sums(S.q[:, :1, :K - 1], S.q[:, :1, :K - 1])[0, 0, 0] == 2 ** 31 - 4096
    # stage 1: the mantissa digits (up to 127) of the tensor against balanced digits of the right factor
    assert M.int32_ok(7, 37744, 127, 64) and not M.int32_ok(7, 37745, 127, 64)


@pytest.mark.parametrize('kb_per', [1, 2])
def test_stage2_ranges_and_symmetry(kb_per):
    """K ranges change the result only by fp64 re-association; the symmetric mode keeps the upper triangle."""
    rng = np.random.RandomState(kb_per)
    A = rng.standard_normal((40, 300))
    B = A + 1e-3 * rng.standard_normal((40, 300))
    Sa, Sb = M.slice_rows(A, 7), M.slice_rows(B, 7)
    C1, _ = M.stage2(Sa, Sb)
    C2, parts = M.stage2(Sa, Sb, kb_per=kb_per)
    assert len(parts) == -(-Sa.Kp // (128 * kb_per))
    assert (np.abs(C1 - C2) <= M.ranges_bound(parts) + 2.0 ** -52 * np.abs(C1)).all()
    Cs, _ = M.stage2(Sa, Sb, symmetric=True)
    assert (Cs == np.triu(C1)).all()
    ref = M.exact_abt(A, B)
    assert (np.abs(C1 - ref) <= M.product_bound(7, 300, Sa.E[:40], Sb.E[:40])).all()


# ------------------------------------------------------------------------------------------------- DF-K through the model
def model_df_k(cderi, nao, dm, ns, occ=None, hermi=0):
    """K of df.cu's int8 engine computed by the model, block = all rows: (K, bound).  occ: orbitals C~ [nao][nocc] (tagged
    path, K = Y Y^T); else the general density (K = Y G^T, G[l][(P, k)] = A_P[l][k]).  Y is cut by the fused epilogue with
    the Cauchy-Schwarz exponent bound from float32 row norms, as yexp_bound_kernel computes it."""
    nr = cderi.shape[0]
    SA, _ = M.slice_packed(cderi, nao, ns)
    X = M.unpack_rows(cderi, nao)
    right = occ.T.copy() if occ is not None else dm.T.copy()           # rows [ncol][nao]
    ncol = right.shape[0]
    SC = M.slice_rows(right, ns)
    ncolp = M.pad_to(ncol, 16)
    rn2 = (X.astype(np.float64) ** 2).astype(np.float32).reshape(nr, nao, nao).sum(axis=2, dtype=np.float32)
    cmax2 = (right ** 2).sum(axis=1).max()
    bound = 1.001 * np.sqrt(rn2.max(axis=0).astype(np.float64) * 1.0001 * cmax2)
    Ey = np.where(bound > 0, M.frexp_exp(np.where(bound > 0, bound, 1.0)), 0)
    SY = M.stage1_y(SA, SC, Ey, 0, nr * nao, nao, ncolp)
    # exact Y, and the bound of the Y the digits represent against it
    Yex = np.einsum('pab,bi->api', X.reshape(nr, nao, nao), right.T).reshape(nao, nr * ncol)
    Yq = M.reconstruct(SY.q[:, :nao, :SY.K], Ey).reshape(nao, nr, ncolp)[:, :, :ncol].reshape(nao, nr * ncol)
    assert (np.abs(Yex) < np.ldexp(1.0, Ey.astype(np.int32))[:, None]).all(), 'Ey is not a bound'
    dY = M.product_bound(ns, nao, SA.E[:nr * nao], SC.E[:ncol], SA.dmax, 64).reshape(nr, nao, ncol).transpose(1, 0, 2)
    dY = dY.reshape(nao, nr * ncol) + np.ldexp(M.tail_bound(ns), Ey.astype(np.int32))[:, None]
    assert (np.abs(Yq - Yex) <= dY).all()
    if occ is not None:
        SB, Bex, dB = SY, Yex, dY
    else:
        gcol = M.pad_to(nao, 16)
        G = np.zeros((nao, nr, gcol))
        G[:, :, :nao] = X.reshape(nr, nao, nao).transpose(1, 0, 2)
        SB = M.slice_rows(G.reshape(nao, nr * gcol), ns)
        Bex, dB = X.reshape(nr, nao, nao).transpose(1, 0, 2).reshape(nao, nr * nao), 0.0
    K, _ = M.stage2(SY, SB, symmetric=(occ is not None or hermi == 1))
    if occ is not None or hermi == 1:
        K = np.triu(K) + np.triu(K, 1).T
    # bound: error of the Y digits carried through K = Y B^T, plus stage 2's own slicing (Y digits are exact inputs there)
    Kb = dY @ np.abs(Bex).T + np.abs(Yq) @ (dB if np.ndim(dB) else np.zeros_like(Bex)).T
    Kb += M.product_bound(ns, SY.K, SY.E[:nao], SB.E[:nao], 64, 64)
    return K, Kb


def _df_case(name):
    from pyscf_b200 import gto
    from pyscf_b200.gto.mole import make_auxmol
    from oracle import oracle as O
    if name == 'h2o':
        mol = gto.M(atom='O 0 0 0; H 0 -0.757 0.587; H 0 0.757 0.587', basis='cc-pvdz')
        aux = 'weigend'
    else:
        mol = gto.M(atom='He 0 0 0; Ne 1.2 0.3 0', basis='cc-pvtz')        # f orbital shells, g auxiliary shells
        aux = 'def2-universal-jkfit'
    cderi, nao = O.cholesky_eri(mol, make_auxmol(mol, aux))
    return cderi, nao, O


_MARGIN = {}


@pytest.mark.parametrize('name', ['h2o', 'hene'])
@pytest.mark.parametrize('ns', [5, 6, 7, 8])
@pytest.mark.parametrize('kind', ['tagged', 'general0', 'general1'])
def test_df_k_model_against_oracle(name, ns, kind):
    """The engine's DF-K algorithm (packed tensor slices, fused Y with its Cauchy-Schwarz exponents, stage 2 in symmetric or
    full mode) run through the model equals the oracle's FP64 K within the model-derived bound.  With 7 slices the bound
    stays below the 1e-9 bar of the DF tests."""
    cderi, nao, O = _df_case(name)
    rng = np.random.RandomState(ns)
    c = np.linalg.qr(rng.standard_normal((nao, 5)))[0] * np.sqrt(2.0)
    if kind == 'tagged':
        dm = c @ c.T
        K, Kb = model_df_k(cderi, nao, dm, ns, occ=c)
    else:
        dm = rng.random_sample((nao, nao))
        if kind == 'general1':
            dm = dm + dm.T
        K, Kb = model_df_k(cderi, nao, dm, ns, hermi=int(kind == 'general1'))
    ref = O.df_get_jk(cderi, nao, dm)[1]
    err = np.abs(K - ref)
    tol = Kb + 1e-13 * np.abs(ref).max()                                  # the oracle's own fp64 rounding
    assert (err <= tol).all(), (err.max(), tol.max())
    if ns == 7:
        # observed error at least 10x under the 1e-9 bar; the worst-case bound is under it for the tagged path only
        # (general densities: ~1e-8, the bound multiplies by sum |G| over all (P, k))
        assert err.max() < 1e-10
        assert kind != 'tagged' or Kb.max() < 1e-9, Kb.max()
