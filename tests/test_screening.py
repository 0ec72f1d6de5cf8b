"""The on-device screening of the 4-center J/K path, quartet by quartet, against tests/screen_ref.py.

Every other accuracy test of the direct path runs with the screening off or with a dense random density, where all six
density terms of the prescreen give the same answer.  Here the densities are block-sparse and spread over many decades, the
tolerances are the production 1e-13 and the loose 1e-9 and 1e-6 (where a wrongly dropped quartet is worth far more than the
bar), and the expected J/K are the long-double integrals digested over exactly the quartets the rule keeps.

Bar per output element: |kernel - expected| <= KAPPA eps sum S|D| + sum over ambiguous quartets of S|D| (KAPPA = 1024 as in
tests/test_rys_eri.py, and as there S is the largest S_abs of the element's shell-quartet block); an element whose sums are
empty must be exactly 0.  Counters: quartets_computed within the bounds the ambiguous quartets leave, computed + screened
equal to the number of unique pair-list quartets, exactly.  The dm_cond table (b200jk_get_dm_cond_test) is compared bit for
bit.

Systems (centres dyadic in bohr):
* chain: four atoms on a line, 2.5 to 4 bohr apart, twelve one-primitive shells (each of s, p, d, f on three of the atoms)
  with exponents 0.25 to 5; q runs from O(1) to below 1e-14 and all 55 classes keep and drop quartets.
* segments: a 5-primitive d shell (25 primitive pairs: list entries of 16 + 9) and nctr = 2 d and f shells, 6 bohr apart.
* slattice: 48 s shells and 16 d shells on a distorted 4 x 4 x 3 lattice.  Its 136 (dd| bra pairs outnumber the SMs, so with
  B200JK_WANT_CTAS=1 every (dd|ss) block-kernel CTA gets the whole (ss| list (more than 512 entries at every tolerance, more
  than 1024 at 1e-13) and walks it in sub-chunks of the 512-entry shared list.
"""
import os
import re
import subprocess
import sys
import time

import numpy as np
import pytest

import eri_ref as R
import screen_ref as S
from screen_ref import TOLS, decade_density, golden_cases, one_sided_density
from test_rys_eri import ALL_CLASSES, BAR, HE, KAPPA, NE, PAIR_ID, class_name, family, launched
from pyscf_b200 import gto
from pyscf_b200 import lib as b2lib
from pyscf_b200.jk import VHFOpt

pytestmark = pytest.mark.skipif(not R.LONGDOUBLE_OK, reason=R.SKIP_REASON)

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
MAX_AMBIGUOUS = 4          # unique segment quartets per call; measured: 0 in every case below

SYSTEMS = {
    'chain': S.CHAIN,
    'segments': dict(atom='Ne 0 0 0; He 0 0 6', basis={'Ne': [[0, [30., 0.2], [5., 0.5], [0.8, 0.5]], NE[2]],
                                                        'He': [[1, [0.9, 1.0]], HE[1], HE[2]]}),
}


# ---------------------------------------------------------------------------------------------------------------------
class Case:
    """A system with one operator and AO convention: the model's basis, integrals and q, and the library's orientation of
    every unique cross-class quartet (for the coverage counts)."""

    def __init__(self, name, omega, cart):
        t = time.time()
        self.name, self.omega, self.cart = name, omega, cart
        self.mol = gto.M(unit='Bohr', cart=cart, **SYSTEMS[name])
        self.basis = B = S.Basis(self.mol._atm, self.mol._bas, self.mol._env, cart)
        self.eri, self.sab, self.q = B.integrals(omega)
        # the scale of an element is the largest S_abs of its shell-quartet block, as in tests/test_rys_eri.py
        blk = self.sab
        for ax in range(4):
            blk = np.maximum.reduceat(blk, B.off[:-1], axis=ax)
        s = B.seg_of_ao
        self.sab = blk[np.ix_(s, s, s, s)]
        self.seconds = time.time() - t
        a, b = S.unique_pairs(B.nseg)
        rank = np.argsort(B.dev)                        # segment -> device shell
        swap = rank[a] < rank[b]
        self.pi, self.pj = np.where(swap, b, a), np.where(swap, a, b)      # device order: ish >= jsh
        self.pcls = PAIR_ID(B.ls[a], B.ls[b])
        P, Q = np.meshgrid(np.arange(len(a)), np.arange(len(a)), indexing='ij')
        cls = [launched(int(x), int(y)) for x, y in zip(self.pcls[P].ravel(), self.pcls[Q].ravel())]
        bra_ok = np.array([c[0] for c in cls]).reshape(P.shape) == self.pcls[P]
        sel = (self.pcls[P] != self.pcls[Q]) & bra_ok
        self.obra, self.oket = P[sel], Q[sel]
        self.ocls = [c for c, s in zip(cls, sel.ravel()) if s]
        self.ofam = np.array([family(c) for c in self.ocls])

    def oriented(self, m4):
        """A [nseg]*4 array at (ish, jsh, ksh, lsh) of every unique cross-class quartet as the library launches it."""
        return m4[self.pi[self.obra], self.pj[self.obra], self.pi[self.oket], self.pj[self.oket]]


_CASES = {}


def case(name, omega=0.0, cart=False):
    key = (name, omega, cart)
    if key not in _CASES:
        _CASES[key] = Case(*key)
        print('reference %s omega=%g%s: %.0f s' % (name, omega, ' cart' if cart else '', _CASES[key].seconds), flush=True)
    return _CASES[key]


# ---------------------------------------------------------------------------------------------------------------------
# densities
def blocks(B, a, b):
    return slice(B.off[a], B.off[a + 1]), slice(B.off[b], B.off[b + 1])


def probe_density(B, a, b, m, sym=True, seed=0):
    """Nonzero in the segment block (a, b) only (and its transpose): values in [m/2, m], the largest exactly m."""
    rng = np.random.RandomState(seed)
    d = np.zeros((B.nao, B.nao))
    sa, sb = blocks(B, a, b)
    blk = m * (0.5 + 0.5 * rng.random_sample((sa.stop - sa.start, sb.stop - sb.start))) * rng.choice([-1.0, 1.0])
    blk.flat[0] = m
    d[sa, sb] = blk
    if a == b:
        d[sa, sb] = 0.5 * (blk + blk.T)
        d[sa.start, sb.start] = m
    if sym:
        d[sb, sa] = d[sa, sb].T
    return d


# ---------------------------------------------------------------------------------------------------------------------
class Run:
    """One handle per tolerance of a case; every call is checked in full and tallied."""

    def __init__(self, lib, cs):
        self.lib, self.cs = lib, cs
        self.opts = {}
        self.worst = {}            # family -> largest error / bar (J outputs of the single-block probes)
        self.worst_all = 0.0
        self.n_amb = 0
        self.calls = 0
        self.sole = {}             # (family, term) -> unique quartets kept through that term alone
        self.cls_kept, self.cls_dropped = set(), set()
        self.window = {'tpq': 0, 'block': 0}      # kept through a J term that fails without its factor 4
        self.qq_drop_calls = 0                    # calls with a 1e30 density in which q_ij q_kl <= tol drops quartets

    def opt(self, tol):
        if tol not in self.opts:
            self.opts[tol] = VHFOpt(self.cs.mol, direct_scf_tol=tol, omega=self.cs.omega, libpath=self.lib)
        return self.opts[tol]

    def close(self):
        for o in self.opts.values():
            o.close()

    def dm_cond_table(self, opt):
        h = opt.handle
        nsh = self.cs.basis.nseg
        assert opt.stats()['n_dev_shells'] == nsh
        t = np.zeros((nsh, nsh))
        off = np.zeros(nsh, dtype=np.int32)
        h.check(h.lib.b200jk_get_dm_cond_test(h._h, b2lib.dptr(t), b2lib.iptr(off), nsh), 'b200jk_get_dm_cond_test')
        return t, off

    def check(self, label, dms, hermi, tol, with_j=True, with_k=True, probe=None, zero_guard=False):
        cs, B = self.cs, self.cs.basis
        opt = self.opt(tol)
        dmc = B.dm_cond(dms)
        dec = S.Decision(cs.q, dmc, tol, with_j, with_k, guard=0.0 if zero_guard else S.GUARD)
        vj, vk = opt.get_jk(dms, hermi=hermi, with_j=with_j, with_k=with_k)
        st = opt.stats()
        self.calls += 1
        # the table the kernels screened with, bit for bit, and the device shell order
        got, ao_off = self.dm_cond_table(opt)
        assert np.array_equal(ao_off, B.off[B.dev]), '%s: device shells are not the segments sorted by l' % label
        bad = np.argwhere(got != dmc[np.ix_(B.dev, B.dev)])
        assert not len(bad), '%s: dm_cond differs at device shells %s: %r, expected %r' % (
            label, bad[0], got[tuple(bad[0])], dmc[np.ix_(B.dev, B.dev)][tuple(bad[0])])
        # counters
        ent = B.entries(cs.q, tol)
        qmax = cs.q.max()
        edge = np.abs(cs.q * qmax / (R.LD(tol) * R.LD(S.SETUP_DROP)) - 1)
        assert not (edge < S.GUARD).any(), '%s: a pair sits on the set-up threshold' % label
        total, lo, hi = S.count(None, ent), S.count(dec.lo, ent), S.count(dec.hi, ent)
        n_amb = S.n_unique(dec.amb, B.nseg)
        assert n_amb <= MAX_AMBIGUOUS, '%s: %d ambiguous quartets' % (label, n_amb)
        self.n_amb = max(self.n_amb, n_amb)
        comp, scr = st['quartets_computed'], st['quartets_screened']
        assert comp + scr == total, '%s: computed %d + screened %d != %d unique list quartets' % (label, comp, scr, total)
        assert lo <= comp <= hi, '%s: quartets_computed %d outside [%d, %d]' % (label, comp, lo, hi)
        # J/K over the kept set
        aD = S.abs_density(dms)
        M = S.ao_mask(B, dec.keep)
        ej, ek = S.digest(cs.eri * M, dms, with_j, with_k)
        sj, sk = S.digest(cs.sab * M, aD, with_j, with_k)
        if n_amb:
            aj, ak = S.digest(cs.sab * S.ao_mask(B, dec.amb), aD, with_j, with_k)
        else:
            aj, ak = (0.0 if with_j else None), (0.0 if with_k else None)
        for what, v, e, s, a in (('J', vj, ej, sj, aj), ('K', vk, ek, sk, ak)):
            if v is None:
                continue
            assert np.all(np.isfinite(v)), '%s %s: not finite' % (label, what)
            bar = BAR * s + a
            err = np.abs(v - e)
            ok = np.where(bar > 0, err <= bar, v == 0)
            if not ok.all():
                idx = np.argwhere(~ok)
                i = idx[np.argmax((err / np.where(bar > 0, bar, 1e-300))[~ok])]
                sa, sb = B.seg_of_ao[i[-2]], B.seg_of_ao[i[-1]]
                fed = ''
                if probe is not None and what == 'J':
                    c = launched(int(PAIR_ID(B.ls[probe[0]], B.ls[probe[1]])), int(PAIR_ID(B.ls[sa], B.ls[sb])))
                    fed = ', class %s %s' % (class_name(c), family(c))
                raise AssertionError('%s: %s%s differs in %d elements; worst at %s (segments %d, %d%s): kernel %.17g, '
                                     'expected %.17g, bar %.3g (%d eps x %.3g + ambiguous %.3g)' % (
                                         label, what, list(v.shape), len(idx), tuple(i), sa, sb, fed, v[tuple(i)],
                                         e[tuple(i)], bar[tuple(i)], KAPPA, s[tuple(i)], np.broadcast_to(a, v.shape)[tuple(i)]))
            with np.errstate(divide='ignore', invalid='ignore'):
                ratio = np.where(bar > 0, err / np.where(bar > 0, bar, 1), 0.0)
            self.worst_all = max(self.worst_all, float(ratio.max()))
            if probe is not None and what == 'J':
                rb = np.maximum.reduceat(np.maximum.reduceat(ratio.reshape(-1, B.nao, B.nao).max(axis=0), B.off[:-1], 0),
                                         B.off[:-1], 1)
                pc = int(PAIR_ID(B.ls[probe[0]], B.ls[probe[1]]))
                for sa in range(B.nseg):
                    for sb in range(sa + 1):
                        f = family(launched(pc, int(PAIR_ID(B.ls[sa], B.ls[sb]))))
                        self.worst[f] = max(self.worst.get(f, 0.0), float(rb[sa, sb]))
        self.cover(dec, dmc, tol, with_j)
        return dec, st

    def cover(self, dec, dmc, tol, with_j):
        """Coverage bookkeeping of one call, over the unique quartets in the library's orientation."""
        cs, B = self.cs, self.cs.basis
        keep_o = cs.oriented(dec.keep)
        for t in S.TERMS:
            so = cs.oriented(dec.sole(t))
            for f in ('tpq', 'block'):
                self.sole[f, t] = self.sole.get((f, t), 0) + int((so & (cs.ofam == f)).sum())
        for c, k in zip(cs.ocls, keep_o):
            (self.cls_kept if k else self.cls_dropped).add(c)
        a, b = S.unique_pairs(B.nseg)
        same = dec.keep[a, b, a, b]
        for c, k in zip(cs.pcls, same):
            (self.cls_kept if k else self.cls_dropped).add((int(c), int(c)))
        if with_j:
            # kept only through J terms, none of which would pass without the factor 4
            d = np.asarray(dmc).astype(R.LD)
            nof = ((d[:, :, None, None] * dec.qq > R.LD(tol)) | (d[None, None, :, :] * dec.qq > R.LD(tol)))
            only_j = dec.keep & ~(dec.passes['jk'] | dec.passes['jl'] | dec.passes['ik'] | dec.passes['il']) & ~nof
            wo = cs.oriented(only_j)
            for f in ('tpq', 'block'):
                self.window[f] += int((wo & (cs.ofam == f)).sum())
        self.qq_drop_calls += int(dmc.max() > 1e20 and bool((dec.qq <= R.LD(tol)).any()))

    def report(self, what):
        print('%s: %d calls, reference %.0f s; largest error / bar %.3f overall, per family (J of the single-block probes) %s; '
              'most ambiguous quartets in one call %d' % (what, self.calls, self.cs.seconds, self.worst_all,
                                                          {k: round(v, 3) for k, v in self.worst.items()}, self.n_amb), flush=True)


# ---------------------------------------------------------------------------------------------------------------------
def probe_magnitude(cs, a, b, tol, k):
    """A block magnitude m for which thresholds tol / qq of the quartets that address (a, b) fall between m and 4 m: m times
    q_ab q_kl = tol / 2 for the k-th pair (k, l) in descending q."""
    qs = np.sort(np.asarray(cs.q[np.tril_indices(cs.basis.nseg)], dtype=np.float64))[::-1]
    qs = qs[qs > 0]
    return float(tol / 2 / (float(cs.q[a, b]) * qs[min(k, len(qs) - 1)]))


def chain_probes(run, stride=1, tols=TOLS):
    """Single-block probes over the segment blocks of the chain."""
    cs, B = run.cs, run.cs.basis
    a, b = S.unique_pairs(B.nseg)
    n = 0
    for pa, pb in list(zip(a, b))[::stride]:
        if cs.q[pa, pb] < 1e-12:
            continue
        for it, tol in enumerate(tols):
            m = probe_magnitude(cs, pa, pb, tol, 5 + 7 * ((n + it) % 9))
            mode = (n + it) % 4
            lab = 'chain probe block (%d, %d) m = %.3g tol %g' % (pa, pb, m, tol)
            if mode == 0:
                run.check(lab, probe_density(B, pa, pb, m, seed=n), 1, tol, probe=(pa, pb))
            elif mode == 1:
                run.check(lab + ' K only', probe_density(B, pa, pb, m, seed=n), 1, tol, with_j=False)
            elif mode == 2:
                run.check(lab + ' J only', probe_density(B, pa, pb, m, seed=n), 1, tol, with_k=False, probe=(pa, pb))
            else:
                run.check(lab + ' one-sided', probe_density(B, pa, pb, 2 * m, sym=False, seed=n), 0, tol, probe=(pa, pb))
        n += 1


def chain_densities(run, tols=TOLS):
    cs, B = run.cs, run.cs.basis
    for tol in tols:
        dd = decade_density(B, 11)
        dec_jk, _ = run.check('chain decade tol %g' % tol, dd, 1, tol)
        dec_j, _ = run.check('chain decade J only tol %g' % tol, dd, 1, tol, with_k=False)
        dec_k, _ = run.check('chain decade K only tol %g' % tol, dd, 1, tol, with_j=False)
        # the kept sets differ as the rule says: J and K sets unite to the J+K set, neither contains the other
        assert np.array_equal(dec_j.keep | dec_k.keep, dec_jk.keep)
        assert (dec_j.keep & ~dec_k.keep).any() and (dec_k.keep & ~dec_j.keep).any()
        run.check('chain one-sided tol %g' % tol, one_sided_density(B, 12), 0, tol)
        anti = decade_density(B, 13, sym=False)
        run.check('chain antisymmetric tol %g' % tol, anti - anti.T, 2, tol)
        # a batch whose blocks are large in different densities
        batch = np.array([decade_density(B, s) for s in (21, 22, 23)])
        dmc1 = [B.dm_cond(d) for d in batch]
        assert all((B.dm_cond(batch) > d).any() for d in dmc1)
        dec_b, _ = run.check('chain batch of 3 tol %g' % tol, batch, 1, tol)
        assert all((dec_b.keep & ~S.Decision(cs.q, d, tol).keep).any() for d in dmc1)
        run.check('chain batch of 3, one-sided tol %g' % tol, np.array([one_sided_density(B, s) for s in (31, 32, 33)]), 0, tol)
        # nothing and everything
        dec0, st = run.check('chain zero density tol %g' % tol, np.zeros((B.nao, B.nao)), 1, tol)
        assert st['quartets_computed'] == 0 and not dec0.keep.any()
        dech, _ = run.check('chain huge density tol %g' % tol, decade_density(B, 14, kmax=0) * 1e30, 1, tol)
        assert np.array_equal(dech.keep, dech.qq > R.LD(tol)) and not dech.keep.all()


def chain_coverage(run):
    for f in ('tpq', 'block'):
        for t in S.TERMS:
            assert run.sole.get((f, t), 0) > 0, 'no %s quartet kept through d_%s alone: %s' % (f, t, run.sole)
        assert run.window[f] > 0, 'no %s quartet kept only by the factor 4 of a J term' % f
    assert run.qq_drop_calls > 0
    missing = [class_name(c) for c in ALL_CLASSES if c not in run.cls_kept or c not in run.cls_dropped]
    assert not missing, 'classes without both kept and dropped quartets: %s' % missing
    print('quartets kept through one term alone, per family:', run.sole, 'factor-4 window:', run.window, flush=True)


def run_chain(lib, omega=0.0, cart=False, stride=1, dens=True, what='chain'):
    cs = case('chain', omega, cart)
    assert float(cs.q.max()) > 0.5 and float(cs.q[cs.basis.nprim > 0].min()) < 1e-14
    run = Run(lib, cs)
    t = time.time()
    chain_probes(run, stride)
    if dens:
        chain_densities(run)
    if stride == 1 and dens:
        chain_coverage(run)
    run.report('%s omega=%g%s (%.0f s)' % (what, omega, ' cart' if cart else '', time.time() - t))
    run.close()
    return run


# ---------------------------------------------------------------------------------------------------------------------
# the model against things that are not the model
def test_constants_match_kernel_sources():
    src = os.path.join(ROOT, 'pyscf_b200', 'csrc')
    core = open(os.path.join(src, 'jk_core.cuh')).read()
    assert int(re.search(r'constexpr int MAX_PRIM_PER_PAIR = (\d+);', core).group(1)) == S.MAX_PRIM_PER_PAIR
    host = open(os.path.join(src, 'b200jk.cu')).read()
    assert 'if (!(sp.q * qmax > tol * 1e-2)) continue;' in host and S.SETUP_DROP == 1e-2
    assert 'p0 += MAX_PRIM_PER_PAIR' in host
    common = open(os.path.join(src, 'host_common.hpp')).read()
    assert float(re.search(r'constexpr double PRIM_CUT = ([0-9.e+-]+);', common).group(1)) == R.PRIM_CUT
    assert 'constexpr int KCH_MAX = 512;' in open(os.path.join(src, 'jk_block.cuh')).read()


def model_jk(cs, dm, tol):
    B = cs.basis
    dec = S.Decision(cs.q, B.dm_cond(dm), tol)
    M = S.ao_mask(B, dec.keep)
    aD = S.abs_density(dm)
    return dec, S.digest(cs.eri * M, dm), S.digest(cs.sab * M, aD), S.digest(cs.sab * S.ao_mask(B, dec.amb), aD)


def test_model_against_oracle_and_reference_driver():
    """The restated rule against the oracle's screened driver (kept count, J/K) and against the reference's own
    CVHFnrs8_prescreen / CVHFnr_dm_cond (stored results, and the live routine where oracle/_ref is built)."""
    from oracle import oracle as O
    from oracle import ref_driver
    cs = case('chain')
    B = cs.basis
    gold = np.load(os.path.join(HERE, 'golden', 'screen_ref.npz'))
    ones = np.ones((B.nseg, B.nseg), dtype=int)
    for name, (dm, hermi) in golden_cases(B).items():
        assert np.array_equal(gold['%s_dm' % name], dm) and int(gold['%s_hermi' % name]) == hermi
        for tol in TOLS:
            dec, (ej, ek), (sj, sk), (aj, ak) = model_jk(cs, dm, tol)
            assert S.n_unique(dec.amb, B.nseg) <= MAX_AMBIGUOUS
            assert 0 < S.n_unique(dec.keep, B.nseg) < S.n_unique(None, B.nseg)
            oj, ok, n = O.get_jk(cs.mol, dm, direct_scf_tol=tol, screen=True, return_count=True)
            assert S.count(dec.lo, ones) <= n <= S.count(dec.hi, ones), (name, tol, n)
            refs = [('oracle', oj, ok), ('stored reference driver', gold['%s_%g_vj' % (name, tol)], gold['%s_%g_vk' % (name, tol)])]
            if ref_driver.available():
                refs.append(('reference driver',) + tuple(ref_driver.get_jk(cs.mol, dm, hermi=hermi, direct_scf_tol=tol)))
            for what, rj, rk in refs:
                for v, e, s, a in ((rj, ej, sj, aj), (rk, ek, sk, ak)):
                    assert np.all(np.abs(v - e) <= BAR * s + a), (what, name, tol, float((np.abs(v - e) / (BAR * s + a + 1e-300)).max()))


# ---------------------------------------------------------------------------------------------------------------------
def check_q_cond(lib, cs, tol=1e-13):
    """b200jk_get_q_cond against the long-double q at 1e-10 relative down to the smallest q, and the 1e-100 floor."""
    B = cs.basis
    opt = VHFOpt(cs.mol, direct_scf_tol=tol, omega=cs.omega, libpath=lib)
    q = opt.q_cond
    opt.close()
    qs, _ = B.per_shell(cs.q, np.zeros((B.nseg, B.nseg)))
    first = np.array([np.argmax(B.shell == s) for s in range(B.shell.max() + 1)])
    qm = qs[first][:, first]
    live = qm > 0
    assert live.any() and (cs.name != 'chain' or float(qm[live].min()) < 1e-14)
    rel = np.abs(q[live] / qm[live].astype(np.float64) - 1)
    assert rel.max() <= 1e-10, '%s: q_cond off by %.3g relative at q = %.3g' % (cs.name, rel.max(), float(qm[live][rel.argmax()]))
    assert np.all(q[~live] == 1e-100)


def test_q_cond_against_long_double(emu_lib):
    for omega in (0.0, 0.35, -0.4):
        check_q_cond(emu_lib, case('chain', omega))
    check_q_cond(emu_lib, case('chain', 0.0, True))
    check_q_cond(emu_lib, case('segments'))
    # a pair without a surviving primitive pair reports the floor exactly
    mol = gto.M(unit='Bohr', atom='H 0 0 0; He 0 0 16', basis={'H': [[0, [40.0, 1.0]]], 'He': [[0, [30.0, 1.0]]]})
    opt = VHFOpt(mol, libpath=emu_lib)
    q = opt.q_cond
    opt.close()
    assert q[0, 1] == 1e-100 and q[1, 0] == 1e-100 and q[0, 0] > 1


def test_chain_emulated(emu_lib):
    """Coulomb operator, spherical AOs: every probe and density, with the coverage assertions."""
    run_chain(emu_lib)


@pytest.mark.parametrize('omega,cart', [(0.35, False), (-0.4, False), (0.0, True)])
def test_chain_operators_and_cartesian_emulated(emu_lib, omega, cart):
    run_chain(emu_lib, omega, cart, stride=5)


def test_chain_probes_experimental_layouts_emulated(emu_lib_experimental):
    run_chain(emu_lib_experimental, stride=3, dens=False, what='chain, experimental layouts')


def test_chain_loose_tolerances_without_guard_band(emu_lib):
    """With the ambiguity band at zero width the 1e-9 and 1e-6 cases still pass: no case rests on the band."""
    cs = case('chain')
    run = Run(emu_lib, cs)
    for tol in (1e-9, 1e-6):
        run.check('decade, no band, tol %g' % tol, decade_density(cs.basis, 11), 1, tol, zero_guard=True)
        run.check('one-sided, no band, tol %g' % tol, one_sided_density(cs.basis, 12), 0, tol, zero_guard=True)
    chain_probes(run, stride=6, tols=(1e-9, 1e-6))
    run.close()


def run_segments(lib):
    cs = case('segments')
    B = cs.basis
    assert {2, 3} <= {int(b[1]) for b in cs.mol._bas if b[3] > 1}                      # nctr = 2 d and f shells
    assert (B.nprim > S.MAX_PRIM_PER_PAIR).any() and B.nseg > len(cs.mol._bas)
    run = Run(lib, cs)
    split = B.entries(cs.q, 1e-13) > 1
    assert split.any()
    seen_split, n_extra, worst_lost = set(), 0, 0.0
    for tol in TOLS:
        for seed, hermi in ((41, 1), (42, 0)):
            dm = decade_density(B, seed) if hermi else one_sided_density(B, seed)
            dec, _ = run.check('segments decade seed %d tol %g' % (seed, tol), dm, hermi, tol)
            # a split pair is one decision for all of its list entries: both outcomes occur (the counters weigh them)
            a, b = np.argwhere(split)[0]
            seen_split |= set(np.unique(dec.keep[a, b]).tolist())
            # per segment against per contracted shell: the segment rule only ever drops more, and the J/K it gives up (the
            # reference integrals digested over the additionally dropped quartets) stays at the scale of tol: each dropped
            # quartet adds at most tol per AO product (Schwarz and the rule, densities below 1), an output element collects
            # at most 49 products from each
            qs, ds = B.per_shell(cs.q, B.dm_cond(dm))
            per_shell = S.Decision(qs, ds, tol)
            assert not (dec.keep & ~per_shell.keep).any()
            extra = per_shell.keep & ~dec.keep
            n = S.n_unique(extra, B.nseg)
            n_extra += n
            if n:
                dj, dk = S.digest(cs.eri * S.ao_mask(B, extra), dm)
                lost = max(np.abs(dj).max(), np.abs(dk).max())
                worst_lost = max(worst_lost, lost / tol)
                assert lost <= 49 * n * tol, 'the per-segment rule gives up %.3g in J/K at tol %g over %d quartets' % (lost, tol, n)
        for k, (a, b) in enumerate(np.argwhere(np.tril(split))):
            m = probe_magnitude(cs, a, b, tol, 3 + 4 * k)
            run.check('segments probe split pair (%d, %d) tol %g' % (a, b, tol), probe_density(B, a, b, m, seed=k), 1, tol, probe=(a, b))
        run.check('segments n_dm = 1 J only tol %g' % tol, decade_density(B, 43), 1, tol, with_k=False)
    assert seen_split == {False, True} and n_extra > 0
    print('segments: %d quartets dropped per segment that the per-shell rule keeps; largest J/K element they are worth: %.3g tol'
          % (n_extra, worst_lost))
    run.report('segments')
    run.close()


def test_segments_emulated(emu_lib):
    run_segments(emu_lib)


# ---------------------------------------------------------------------------------------------------------------------
S_EXPS = (0.2, 0.7, 2.5, 1.8, 0.35, 0.5, 1.3)
D_EXPS = (0.2, 0.3, 0.45, 0.6, 0.8)
SM_COUNT = 132             # SMs of an H100; the emulation's device_sm_count() returns the same number
KCH_MAX = 512


def slattice_system():
    """48 sites of a 4 x 4 x 3 lattice of spacing 1.5 bohr, each moved off its site by a few dyadic fractions so that no two
    pairs are equivalent by symmetry; an s shell on every site and a d shell on every third one (16 d shells, 136 (dd| pairs)."""
    atoms, basis = [], {}
    n = 0
    for x in range(4):
        for y in range(4):
            for z in range(3):
                lab = 'H%d' % n
                basis[lab] = [[0, [S_EXPS[n % 7], 1.0]]] + ([[2, [D_EXPS[(n // 3) % 5], 1.0]]] if n % 3 == 0 else [])
                atoms.append('%s %r %r %r' % (lab, 1.5 * x + 0.125 * (3 * n % 5), 1.5 * y + 0.125 * (5 * n % 7),
                                              1.5 * z + 0.0625 * (7 * n % 3)))
                n += 1
    return dict(atom='; '.join(atoms), basis=basis)


class SLattice:
    """The lattice's model at the level of shell pairs (its AO tensor would have 128^4 elements): q of every pair, the
    (ss|ss) integrals in closed form and the (dd|ss) blocks from eri_ref's formulas taken over all pairs at once.  Only J is
    built, from densities confined to the s-s block, so the kept quartets are decided by 4 d_kl of an (ss| pair alone and the
    s-s and d-d blocks of J need no other integrals."""

    def __init__(self):
        t = time.time()
        self.mol = gto.M(unit='Bohr', **slattice_system())
        self.basis = B = S.Basis(self.mol._atm, self.mol._bas, self.mol._env)
        self.a, self.b = S.unique_pairs(B.nseg)
        la, lb = B.ls[self.a], B.ls[self.b]
        live = np.array([B.ref.pairs[k].nprim > 0 for k in zip(self.a, self.b)])
        self.ss = np.flatnonzero((la == 0) & (lb == 0) & live)
        self.dd = np.flatnonzero((la == 2) & (lb == 2) & live)
        obj = lambda idx: [B.ref.pairs[self.a[p], self.b[p]] for p in idx]
        self.vss, _ = S.ssss_closed_form(obj(self.ss), obj(self.ss))
        v, sab = S.batched_quartets(obj(self.dd), obj(self.ss))
        for i, j in ((0, 0), (len(self.dd) // 2, 7), (len(self.dd) - 1, len(self.ss) - 1)):       # against the general code
            bra, ket = obj(self.dd[[i]])[0], obj(self.ss[[j]])[0]
            ref = R.quartet(bra, ket)[0]
            assert np.abs(v[i, j] - ref).max() <= 64 * np.finfo(R.LD).eps * np.abs(ref).max(), (i, j)
            ref = R.quartet(ket, ket)[0][0, 0]
            assert abs(self.vss[j, j] - ref) <= 64 * np.finfo(R.LD).eps * abs(ref), j
        T = B.T[2]
        shp = (len(self.dd), len(self.ss), 6, 6)
        self.vdd = np.einsum('ma,bkac,nc->bkmn', T, v.reshape(shp), T).astype(np.float64)
        self.sdd = np.einsum('ma,bkac,nc->bkmn', np.abs(T), sab.reshape(shp), np.abs(T)).astype(np.float64).max(axis=(2, 3))
        self.qp = np.zeros(len(self.a), dtype=R.LD)
        self.qp[self.ss] = np.sqrt(np.abs(self.vss.diagonal()))
        for p in np.flatnonzero(((la == 2) | (lb == 2)) & live):                                  # (ds| and (dd| pairs
            pr = B.ref.pairs[self.a[p], self.b[p]]
            ls = (pr.la, pr.lb, pr.la, pr.lb)
            blk = B._to_ao(R.quartet(pr, pr)[0].reshape([R.ncart(l) for l in ls]), ls, B.T)
            n = blk.shape[0] * blk.shape[1]
            self.qp[p] = np.sqrt(np.abs(blk.reshape(n, n).diagonal()).max())
        self.vss = self.vss.astype(np.float64)
        self.q = np.zeros((B.nseg, B.nseg), dtype=R.LD)
        self.q[self.a, self.b] = self.q[self.b, self.a] = self.qp
        self.seconds = time.time() - t

    def density(self, seed, kmax):
        B = self.basis
        d = decade_density(B, seed, kmax=kmax)
        s = B.ls[B.seg_of_ao]
        d[(s[:, None] != 0) | (s[None, :] != 0)] = 0.0
        return d


def slattice_partition(sl, tol, sm_count):
    """The ket range of every (dd|ss) CTA as the library cuts it: the (ss| list in descending q, kchunk from pick_kchunk.
    Returns (positions of the model's (ss| pairs in the list, kchunk)."""
    B = sl.basis
    ent = B.entries(sl.q, tol)[sl.a, sl.b]
    kets = sl.ss[ent[sl.ss] > 0]
    qk = np.asarray(sl.qp[kets], dtype=np.float64)
    order = np.argsort(-qk, kind='stable')
    nbra, nket = int(ent[sl.dd].sum()), len(kets)
    kchunk = S.pick_kchunk(nbra, nket, 1, sm_count, 1)
    # the library sorts its own double-precision q: the members of a sub-chunk are the model's as long as no two q are
    # closer than the guard band across a sub-chunk boundary
    qs = qk[order]
    for c in range(KCH_MAX, nket, KCH_MAX):
        assert qs[c - 1] > qs[c] * (1 + 1e-9), 'q of the kets on either side of list position %d coincide' % c
    return kets[order], kchunk


def test_kchunk_matches_kernel_sources():
    cls = open(os.path.join(ROOT, 'pyscf_b200', 'csrc', 'jk_classes.cuh')).read()
    for line in ('long want_ctas = device_sm_count() * (want_env > 0 ? want_env : B2_WANT_CTAS);', 'long ny = (want_ctas + nbra - 1) / nbra;',
                 'long kc = (nket + ny - 1) / ny;', 'if (kc < unit) kc = unit;', 'return old_cap ? round1_cap : (1 << 30);',
                 'P.kchunk = pick_kchunk(nbx, P.nket, Cfg::GC::NSLOT, kets_cap(KCH_MAX));', 'return %d;' % SM_COUNT):
        assert line in cls, line
    blk = open(os.path.join(ROOT, 'pyscf_b200', 'csrc', 'jk_block.cuh')).read()
    assert 'constexpr int KCH_MAX = %d;' % KCH_MAX in blk and 'const int kbeg = by * P.kchunk;' in blk
    assert 'for (int sub = kbeg; sub < kend; sub += KCH_MAX) {' in blk
    assert S.pick_kchunk(3, 1176, 16, 132, 1) == 27 and S.pick_kchunk(136, 1100, 16, 132, 1) == 1100
    assert family(launched(int(PAIR_ID(2, 2)), 0)) == 'block'


def run_slattice(lib):
    """Called in a process of its own with B200JK_WANT_CTAS=1.  With 136 (dd| bra pairs, more than the 132 SMs, pick_kchunk
    gives every (dd|ss) CTA the whole (ss| list, which it walks in sub-chunks of KCH_MAX: screen, compact into the shared
    list, process, reset, next.  J only, n_dm = 1 (the J[ij] block stays in registers across the sub-chunks) and 2."""
    assert os.environ.get('B200JK_WANT_CTAS') == '1' and 'B200JK_KETS_CAP' not in os.environ
    sm_count = SM_COUNT
    if lib is None:
        import torch
        sm_count = torch.cuda.get_device_properties(0).multi_processor_count
    sl = SLattice()
    B = sl.basis
    print('reference slattice: %.0f s; %d (dd| pairs, %d (ss| pairs' % (sl.seconds, len(sl.dd), len(sl.ss)), flush=True)
    assert len(sl.dd) >= sm_count
    fs = B.off[:-1]                                             # first AO of every segment
    kinds, most_sub, worst, n_amb_max = set(), 0, 0.0, 0
    for tol, seeds, kmax, scale in ((1e-13, (53,), 12, 1.0), (1e-9, (52,), 8, 1.0), (1e-6, (51, 55), 4, 1.0), (1e-6, (54,), 0, 1.0),
                                    (1e-13, (56,), 0, 1.0), (1e-6, (57,), 2, 2.0 ** -24)):
        dms = scale * np.array([sl.density(sd, kmax) for sd in seeds])
        dmc = B.dm_cond(dms)
        dp = dmc[sl.a, sl.b]
        keep, lo, hi = S.decide_pairs_j(sl.qp, dp, tol)
        opt = VHFOpt(sl.mol, direct_scf_tol=tol, libpath=lib)
        vj, _ = opt.get_jk(dms if len(seeds) > 1 else dms[0], hermi=1, with_k=False)
        vj = vj.reshape(dms.shape)
        st = opt.stats()
        opt.close()
        label = 'slattice tol %g seeds %s' % (tol, seeds)
        # counters over every class of the system
        ent = B.entries(sl.q, tol)[sl.a, sl.b]
        edge = np.abs(sl.qp * sl.qp.max() / (R.LD(tol) * R.LD(S.SETUP_DROP)) - 1)
        assert not (edge < S.GUARD).any()
        n_amb = S.count_pairs(hi & ~lo, np.ones(len(ent), dtype=int))
        assert n_amb <= MAX_AMBIGUOUS, (label, n_amb)
        n_amb_max = max(n_amb_max, n_amb)
        comp, scr = st['quartets_computed'], st['quartets_screened']
        assert comp + scr == S.count_pairs(None, ent), (label, comp, scr)
        assert S.count_pairs(lo, ent) <= comp <= S.count_pairs(hi, ent), (label, comp)
        # the partition of the (ss| list the (dd|ss) CTAs walk
        klist, kchunk = slattice_partition(sl, tol, sm_count)
        nket = len(klist)
        assert kchunk == nket > KCH_MAX, (label, kchunk, nket)         # one CTA per bra pair, kend - kbeg = nket > 512
        most_sub = max(most_sub, -(-nket // KCH_MAX))
        pos = {p: i for i, p in enumerate(klist)}
        for b, pb in enumerate(sl.dd):
            if not ent[pb]:
                continue
            kept = keep[pb, klist]
            for c0 in range(0, nket, KCH_MAX):
                n, k = len(kept[c0:c0 + KCH_MAX]), int(kept[c0:c0 + KCH_MAX].sum())
                kinds.add(('first' if c0 == 0 else 'later', 'full' if k == n else ('empty' if k == 0 else 'partial')))
        # J: w[s, k] is the density weight of ket pair k
        ka, kb = fs[sl.a[sl.ss]], fs[sl.b[sl.ss]]
        w = np.where(ka == kb, dms[:, ka, kb], dms[:, ka, kb] + dms[:, kb, ka])              # [nd, nk]
        amb = (hi & ~lo)
        for what, rows, V, Sc in (('d-d', sl.dd, sl.vdd, sl.sdd[:, :, None, None] + 0 * sl.vdd),
                                  ('s-s', sl.ss, sl.vss[:, :, None, None], np.abs(sl.vss)[:, :, None, None])):
            m = keep[np.ix_(rows, sl.ss)][:, :, None, None]
            ma = amb[np.ix_(rows, sl.ss)][:, :, None, None]
            e = np.einsum('bkmn,sk->sbmn', V * m, w)
            bar = BAR * np.einsum('bkmn,sk->sbmn', Sc * m, np.abs(w)) + np.einsum('bkmn,sk->sbmn', Sc * ma, np.abs(w))
            nf = V.shape[2]
            ia, ib = fs[sl.a[rows]], fs[sl.b[rows]]
            ar = np.arange(nf)
            got = vj[:, (ia[:, None] + ar)[:, :, None], (ib[:, None] + ar)[:, None, :]]       # [nd, nrow, nf, nf]
            got_t = vj[:, (ib[:, None] + ar)[:, None, :], (ia[:, None] + ar)[:, :, None]]
            for g in (got, got_t):
                err = np.abs(g - e)
                ok = np.where(bar > 0, err <= bar, g == 0)
                if not ok.all():
                    i = np.argwhere(~ok)[0]
                    raise AssertionError('%s: J %s block of pair (%d, %d) differs: kernel %.17g expected %.17g bar %.3g' % (
                        label, what, sl.a[rows[i[1]]], sl.b[rows[i[1]]], g[tuple(i)], e[tuple(i)], bar[tuple(i)]))
                worst = max(worst, float((err / np.where(bar > 0, bar, 1))[bar > 0].max(initial=0.0)))
    want = {(c, k) for c in ('first', 'later') for k in ('full', 'empty', 'partial')}
    assert want <= kinds and most_sub >= 3, (sorted(want - kinds), most_sub)
    print('slattice: largest error / bar %.3f, most ambiguous quartets in one call %d, up to %d sub-chunks per CTA' % (
        worst, n_amb_max, most_sub), flush=True)
    print('SLATTICE OK')


def slattice_subprocess(lib):
    code = 'import sys; sys.path[:0] = [%r, %r]; import test_screening as t; t.run_slattice(%r)' % (ROOT, HERE, lib)
    out = subprocess.run([sys.executable, '-c', code], env=dict(os.environ, B200JK_WANT_CTAS='1'), capture_output=True, text=True,
                         timeout=1800)
    print(out.stdout[-3000:])
    assert out.returncode == 0 and 'SLATTICE OK' in out.stdout, out.stdout[-3000:] + out.stderr[-3000:]


def test_slattice_sub_chunks_emulated(emu_lib):
    slattice_subprocess(emu_lib)


# ---------------------------------------------------------------------------------------------------------------------
def run_shards(lib):
    """Two ranks: the partial J/K sum to the expected J/K, the counters to the one-rank counters; on the fitted cost model
    and with a cost table that gives every class whole to one rank."""
    cs = case('chain')
    B = cs.basis
    tol = 1e-9
    dm = np.array([decade_density(B, 61), decade_density(B, 62)])
    dec, (ej, ek), (sj, sk), (aj, ak) = model_jk(cs, dm, tol)
    opt = VHFOpt(cs.mol, direct_scf_tol=tol, libpath=lib)
    h = opt.handle
    opt.get_jk(dm, hermi=1)
    one = opt.stats()
    for table in (None, np.full(100, 1.0)):
        h.check(h.lib.b200jk_set_class_costs(h._h, b2lib.dptr(table), 100 if table is not None else 0), 'b200jk_set_class_costs')
        parts, comp, scr = [], 0, 0
        for r in range(2):
            h.check(h.lib.b200jk_set_shard(h._h, r, 2), 'b200jk_set_shard')
            parts.append(opt.get_jk(dm, hermi=1))
            st = opt.stats()
            assert st['quartets_computed'] > 0
            comp, scr = comp + st['quartets_computed'], scr + st['quartets_screened']
        assert (comp, scr) == (one['quartets_computed'], one['quartets_screened']), (table is not None, comp, scr, one)
        for i, (e, s, a) in enumerate(((ej, sj, aj), (ek, sk, ak))):
            v = parts[0][i] + parts[1][i]
            assert np.all(np.abs(v - e) <= BAR * s + a), ('shards', table is not None, 'JK'[i])
    opt.close()


def test_shards_emulated(emu_lib):
    run_shards(emu_lib)


# ---------------------------------------------------------------------------------------------------------------------
# On the H100: the shared-memory atomicAdd compaction, the warp-shuffle counters and the multi-stream launches exist only
# there.  One process per group.
@pytest.mark.gpu
@pytest.mark.parametrize('group', ['chain', 'chain_erfc', 'chain_cart', 'chain_erfc_cart', 'segments', 'slattice', 'shards'])
def test_screening_device(group):
    if group.startswith('chain'):
        full = group == 'chain'
        run_chain(None, -0.4 if 'erfc' in group else 0.0, 'cart' in group, stride=1 if full else 3, what='H100 chain')
        if full:
            check_q_cond(None, case('chain'))
    elif group == 'segments':
        run_segments(None)
        check_q_cond(None, case('segments'))
    elif group == 'slattice':
        slattice_subprocess(None)
    else:
        run_shards(None)
