"""A model of the direct J/K path's quartet screening, independent of the library and of the oracle.

From libcint-layout tables and tests/eri_ref.py (McMurchie-Davidson in long double) it restates, per device shell (one
segment per shell and contraction column):

* q[a, b] = sqrt(max |(ab|ab)|) in long double over the functions of the handle's AO basis (real-spherical, or libcint's
  Cartesian functions), for the handle's operator, read off the diagonal blocks of the integral tensor;
* dm_cond[a, b] = max over densities and over the block of 0.5 (|D_mn| + |D_nm|), in double with the library's operation
  order (abs, one add, one multiply, max), so it can be compared bit for bit;
* the decision of CVHFnrs8_prescreen (pyscf/lib/vhf/optimizer.c:90-117): keep when q_ij q_kl > tol and any of
  4 d_ij, 4 d_kl (J only), d_jk, d_jl, d_ik, d_il (K only) exceeds tol / (q_ij q_kl).  Every comparison is also taken with
  the threshold moved by a relative GUARD either way: a quartet whose outcome differs between the two is *ambiguous* (the
  library's q comes from a Rys quadrature in double) and may go either way;
* the counters: unique quartets over the library's pair-list entries.  A pair with n > 16 surviving primitive pairs is
  ceil(n / 16) entries, a pair with q * qmax <= tol / 100 is removed when the screening is set up and is none;
* J/K restricted to the kept set, J_kl = sum (M eri)_ijkl D_ji, K_il = sum (M eri)_ijkl D_jk, and the same contraction of
  S_abs with |D_sym| + |D_anti| (what the kernels digest), the scale of the accuracy bar.

The integrals are evaluated in long double and stored rounded to double, and the masked contractions run in double: both
roundings are a few eps of sum S |D| per element, far inside the 1024 eps bar they are used with.
"""
import numpy as np

import eri_ref as R

LD = R.LD
MAX_PRIM_PER_PAIR = 16     # jk_core.cuh
SETUP_DROP = 1e-2          # b200jk_set_screening keeps a pair when q * qmax > tol * SETUP_DROP
GUARD = 1e-9
TERMS = ('ij', 'kl', 'jk', 'jl', 'ik', 'il')


def _nf(l, cart):
    return R.ncart(l) if cart else 2 * l + 1


class Basis:
    """Segments of a basis in the caller's AO order, and the order of the library's device shells."""

    def __init__(self, atm, bas, env, cart=False):
        self.cart = bool(cart)
        self.ref = R.Reference(atm, bas, env)
        self.segs = self.ref.segs
        self.nseg = len(self.segs)
        self.ls = np.array([s.l for s in self.segs])
        self.off = np.cumsum([0] + [_nf(l, cart) for l in self.ls])
        self.nao = int(self.off[-1])
        self.seg_of_ao = np.searchsorted(self.off, np.arange(self.nao), side='right') - 1
        self.dev = np.argsort(self.ls, kind='stable')          # device shell -> segment (sorted by l, stable)
        self.shell = np.concatenate([[ib] * int(b[3]) for ib, b in enumerate(np.asarray(bas).reshape(-1, R.BAS_SLOTS))])
        self.nprim = np.zeros((self.nseg, self.nseg), dtype=int)
        for (i, j), p in self.ref.pairs.items():
            self.nprim[i, j] = self.nprim[j, i] = p.nprim
        self.T = [np.eye(R.ncart(l), dtype=LD) if cart else R.c2s_matrix(l) for l in range(4)]

    def _to_ao(self, v, ls, T):
        for ax, l in enumerate(ls):
            v = np.moveaxis(np.tensordot(T[l], v, axes=([1], [ax])), 0, ax)
        return v

    def integrals(self, omega, quartet=R.quartet, skip=None):
        """(eri, S_abs, q): the tensors in the handle's AO basis as doubles, q[nseg, nseg] in long double.  `skip(bra, ket)`
        leaves a block of pair objects out (zeros); `quartet` is the block evaluator."""
        n = self.nao
        eri, sab = np.zeros((n,) * 4), np.zeros((n,) * 4)
        q = np.zeros((self.nseg, self.nseg), dtype=LD)
        Ta = [np.abs(t) for t in self.T]
        keys = sorted(self.ref.pairs)
        for ib, kb in enumerate(keys):
            for kk in keys[:ib + 1]:
                bra, ket = self.ref.pairs[kb], self.ref.pairs[kk]
                if skip is not None and skip(bra, ket):
                    continue
                v, s, _ = quartet(bra, ket, omega)
                ls = (bra.la, bra.lb, ket.la, ket.lb)
                shp = tuple(R.ncart(l) for l in ls)
                v = self._to_ao(v.reshape(shp), ls, self.T)
                s = self._to_ao(s.astype(LD).reshape(shp), ls, Ta).astype(np.float64)
                if kb == kk:
                    na, nb = v.shape[:2]
                    d = np.abs(v.reshape(na * nb, na * nb).diagonal()).max()
                    q[kb[0], kb[1]] = q[kb[1], kb[0]] = np.sqrt(d)
                v = v.astype(np.float64)
                sa, sb, sc, sd = (slice(self.off[x], self.off[x + 1]) for x in (kb[0], kb[1], kk[0], kk[1]))
                for blk, src in ((eri, v), (sab, s)):
                    blk[sa, sb, sc, sd] = src
                    blk[sb, sa, sc, sd] = src.transpose(1, 0, 2, 3)
                    blk[sa, sb, sd, sc] = src.transpose(0, 1, 3, 2)
                    blk[sb, sa, sd, sc] = src.transpose(1, 0, 3, 2)
                    blk[sc, sd, sa, sb] = src.transpose(2, 3, 0, 1)
                    blk[sd, sc, sa, sb] = src.transpose(3, 2, 0, 1)
                    blk[sc, sd, sb, sa] = src.transpose(2, 3, 1, 0)
                    blk[sd, sc, sb, sa] = src.transpose(3, 2, 1, 0)
        return eri, sab, q

    def dm_cond(self, dms):
        """[nseg, nseg] in double, the operations of CVHFnr_dm_cond in order."""
        dms = np.asarray(dms, dtype=np.float64).reshape(-1, self.nao, self.nao)
        a = np.abs(dms)
        v = (0.5 * (a + a.transpose(0, 2, 1))).max(axis=0)
        v = np.maximum.reduceat(v, self.off[:-1], axis=0)
        return np.maximum.reduceat(v, self.off[:-1], axis=1)

    def entries(self, q, tol):
        """Pair-list entries per segment pair: 0 for a pair without primitive pairs or removed at setup."""
        qmax = q.max()
        kept = (self.nprim > 0) & (q * qmax > LD(tol) * LD(SETUP_DROP))
        return np.where(kept, -(-self.nprim // MAX_PRIM_PER_PAIR), 0)

    def per_shell(self, q, dmc):
        """The reference's granularity: maxima over the segments of each contracted shell, spread back over the segments."""
        out = []
        for t in (q, dmc):
            m = np.zeros((self.shell.max() + 1,) * 2, dtype=t.dtype)
            np.maximum.at(m, (self.shell[:, None], self.shell[None, :]), t)
            out.append(m[self.shell][:, self.shell])
        return out


class Decision:
    """keep / ambiguous / passing terms of every quartet of segments, as [nseg]*4 arrays."""

    def __init__(self, q, dmc, tol, with_j=True, with_k=True, guard=GUARD):
        qq = q[:, :, None, None] * q[None, None, :, :]
        d = np.asarray(dmc).astype(LD)
        one = np.ones_like(qq)
        term = {'ij': 4 * d[:, :, None, None] * one, 'kl': 4 * d[None, None, :, :] * one,
                'jk': d[None, :, :, None] * one, 'jl': d[None, :, None, :] * one,
                'ik': d[:, None, :, None] * one, 'il': d[:, None, None, :] * one}
        on = {t: (with_j if t in ('ij', 'kl') else with_k) for t in TERMS}
        self.qq, self.tol = qq, tol

        def rule(thr):
            ok = qq > thr
            return {t: (ok & (term[t] * qq > thr)) if on[t] else np.zeros(qq.shape, dtype=bool) for t in TERMS}

        self.passes = rule(LD(tol))
        any_ = lambda p: np.logical_or.reduce([p[t] for t in TERMS])
        self.keep = any_(self.passes)
        self.lo = any_(rule(LD(tol) * (1 + LD(guard)))) if guard else self.keep
        self.hi = any_(rule(LD(tol) * (1 - LD(guard)))) if guard else self.keep
        assert not (self.lo & ~self.keep).any() and not (self.keep & ~self.hi).any()
        self.amb = self.hi & ~self.lo
        self.npass = sum(self.passes[t].astype(int) for t in TERMS)

    def sole(self, t):
        return self.passes[t] & (self.npass == 1)


def unique_pairs(nseg):
    a, b = np.tril_indices(nseg)
    return a, b


def count_pairs(m2, e):
    """Unique quartets of pair-list entries inside a symmetric [npair, npair] mask (None: all); e: entries per pair."""
    e = np.asarray(e, dtype=np.int64)
    if m2 is None:
        n = int(e.sum())
        return n * (n + 1) // 2
    off = np.tril(m2, -1)
    return int((off * e[:, None] * e[None, :]).sum() + (m2.diagonal() * e * (e + 1) // 2).sum())


def count(mask4, entries):
    """Unique quartets of pair-list entries inside a symmetric [nseg]*4 mask (None: all of them)."""
    a, b = unique_pairs(entries.shape[0])
    m2 = None if mask4 is None else mask4[a[:, None], b[:, None], a[None, :], b[None, :]]
    return count_pairs(m2, entries[a, b])


def n_unique(mask4, nseg):
    """Unique segment quartets inside a symmetric mask."""
    return count(mask4, np.ones((nseg, nseg), dtype=int))


def ao_mask(basis, mask4):
    s = basis.seg_of_ao
    return mask4[np.ix_(s, s, s, s)]


def digest(t4, dms, with_j=True, with_k=True):
    dms = np.asarray(dms, dtype=np.float64)
    shape = dms.shape
    d3 = dms.reshape((-1,) + shape[-2:])
    vj = np.einsum('ijkl,sji->skl', t4, d3, optimize=True).reshape(shape) if with_j else None
    vk = np.einsum('ijkl,sjk->sil', t4, d3, optimize=True).reshape(shape) if with_k else None
    return vj, vk


def abs_density(dms):
    """|D_sym| + |D_anti|: the two parts the kernels digest separately."""
    dms = np.asarray(dms, dtype=np.float64)
    t = np.swapaxes(dms, -1, -2)
    return np.abs(0.5 * (dms + t)) + np.abs(0.5 * (dms - t))


# ---------------------------------------------------------------------------------------------------------------------
def ssss_closed_form(pa, pb, omega=0.0):
    """(ab|cd) of s-type pair objects in closed form, vectorised in long double: pa, pb are lists of eri_ref pair objects of
    one primitive pair each; returns [len(pa), len(pb)] and, for erfc, the S_abs of the two terms."""
    def gather(ps):
        p = np.array([x.p[0] for x in ps], dtype=LD)
        P = np.array([x.P[0] for x in ps], dtype=LD)
        c = np.array([x.E[0, 0, 0] for x in ps], dtype=LD)
        return p, P, c
    p, P, cp = gather(pa)
    q, Q, cq = gather(pb)
    p, q = p[:, None], q[None, :]
    r2 = ((P[:, None, :] - Q[None, :, :]) ** 2).sum(axis=2)
    alpha = p * q / (p + q)
    pref = 2 * R.PI ** LD(2.5) / (p * q * np.sqrt(p + q)) * cp[:, None] * cq[None, :]

    def one(om):
        a, f = alpha, pref
        if om > 0:
            th = LD(om) ** 2 / (LD(om) ** 2 + alpha)
            a, f = alpha * th, pref * np.sqrt(th)
        return f * R.boys(0, a * r2)[0]
    if omega >= 0:
        v = one(omega)
        return v, np.abs(v)
    vc, ve = one(0.0), one(-omega)
    return vc - ve, np.abs(vc) + np.abs(ve)


def batched_quartets(bras, kets, omega=0.0):
    """Contracted Cartesian blocks of every (bra|ket) of two lists of eri_ref pair objects, each of one primitive pair and of
    one angular class per list: (values [nb, nk, nab, ncd], S_abs) in long double.  eri_ref's formulas (its Hermite
    expansions, R tensor and Boys function), taken over all pairs at once instead of over the primitives of one pair."""
    p = np.array([x.p[0] for x in bras], dtype=LD)[:, None]
    q = np.array([x.p[0] for x in kets], dtype=LD)[None, :]
    P = np.array([x.P[0] for x in bras], dtype=LD)
    Q = np.array([x.P[0] for x in kets], dtype=LD)
    Eb = np.stack([x.E[0] for x in bras])          # [nb, nab, hb]
    Ek = np.stack([x.E[0] for x in kets])          # [nk, ncd, hk]
    nb, nk = len(bras), len(kets)
    Lb, Lk = bras[0].la + bras[0].lb, kets[0].la + kets[0].lb
    PQ = (P[:, None, :] - Q[None, :, :]).reshape(-1, 3)
    alpha0 = (p * q / (p + q)).reshape(-1)
    pref0 = (2 * R.PI ** LD(2.5) / (p * q * np.sqrt(p + q))).reshape(-1)
    idx, sign = R._gather(Lb, Lk)

    def one(om):
        alpha, pref = alpha0, pref0
        if om > 0:
            th = LD(om) ** 2 / (LD(om) ** 2 + alpha0)
            alpha, pref = alpha0 * th, pref0 * np.sqrt(th)
        Rt = R._rtensor(Lb + Lk, alpha, PQ, R.boys(Lb + Lk, alpha * (PQ ** 2).sum(axis=1)))
        Rarr = np.stack([Rt[h] for h in R._herm(Lb + Lk)]) * pref
        M = (Rarr[idx] * sign[:, :, None]).reshape(idx.shape[0], idx.shape[1], nb, nk)
        T = np.einsum('hgbk,kcg->hbkc', M, Ek)
        return np.einsum('bah,hbkc->bkac', Eb, T)
    if omega >= 0:
        v = one(omega)
        return v, np.abs(v)
    vc, ve = one(0.0), one(-omega)
    return vc - ve, np.abs(vc) + np.abs(ve)


def decide_pairs_j(qp, dp, tol, guard=GUARD):
    """The J-only rule over pairs of pairs: (keep, lo, hi) as [npair, npair]; qp long double, dp the dm_cond of each pair."""
    qq = qp[:, None] * qp[None, :]
    t = 4 * np.maximum(dp[:, None], dp[None, :]).astype(LD) * qq
    rule = lambda thr: (qq > thr) & (t > thr)
    return rule(LD(tol)), rule(LD(tol) * (1 + LD(guard))), rule(LD(tol) * (1 - LD(guard)))


def pick_kchunk(nbra, nket, unit, sm_count, want_ctas_per_sm):
    """Kets per CTA of a class launch (pick_kchunk of jk_classes.cuh, without the optional cap)."""
    ny = -(-sm_count * want_ctas_per_sm // nbra)
    return max(-(-nket // ny), unit)


# ---------------------------------------------------------------------------------------------------------------------
# The chain system, its densities and the cases of the stored reference-driver fixture (tests/golden/screen_ref.npz): here, so
# that tools/make_golden_screen.py needs the model only.
TOLS = (1e-13, 1e-9, 1e-6)
CHAIN = dict(atom='H 0 0 0; He 0 0 2.5; Li 0 0 6; Be 0 0 10',
             basis={'H': [[0, [0.4, 1.0]], [1, [1.5, 1.0]], [2, [0.6, 1.0]], [3, [2.0, 1.0]]],
                    'He': [[0, [5.0, 1.0]], [1, [0.3, 1.0]], [2, [2.5, 1.0]]],
                    'Li': [[0, [1.2, 1.0]], [1, [3.5, 1.0]], [3, [0.5, 1.0]]],
                    'Be': [[2, [0.25, 1.0]], [3, [1.0, 1.0]]]})


def decade_density(B, seed, kmax=14, sym=True):
    """Random signs and values, block magnitudes 10^-k with k drawn per segment block."""
    rng = np.random.RandomState(seed)
    d = rng.uniform(0.3, 1.0, (B.nao, B.nao)) * rng.choice([-1.0, 1.0], (B.nao, B.nao))
    k = rng.randint(0, kmax + 1, (B.nseg, B.nseg))
    if sym:
        k = np.minimum(k, k.T)
        d = 0.5 * (d + d.T)
    s = B.seg_of_ao
    return d * 10.0 ** -k[s][:, s]


def one_sided_density(B, seed):
    """hermi = 0: decade-spread, and in about half of the blocks D_mn is kept while D_nm is exactly 0."""
    rng = np.random.RandomState(seed)
    d = decade_density(B, seed, sym=False)
    z = np.triu(rng.random_sample((B.nseg, B.nseg)) < 0.5, 1)
    s = B.seg_of_ao
    d[z[s][:, s]] = 0.0
    return d


def golden_cases(B):
    """name -> (density, hermi) of the fixture, on the Basis of the chain."""
    return {'sym': (decade_density(B, 11), 1), 'one_sided': (one_sided_density(B, 12), 0)}
