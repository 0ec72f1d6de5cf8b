// jk_swq.cuh — "sub-warp per quartet" kernels for the contracted three-root classes whose Cartesian block (54-108 integrals)
// is too large for one thread of jk_tpq.cuh.
//
// A shell quartet gets T consecutive lanes (T = 2, 4 or 8, so a quartet never straddles a warp).  Lane t owns the ket
// Cartesian component pairs cd = t, t + T, ... < NKL, each with the whole bra block in registers (at most 36 accumulators per
// lane, the register budget of the thread-per-quartet kernels).  Every lane evaluates all Rys roots and the vertical recurrence
// of the primitive quartet itself (timed against lanes splitting the roots and exchanging them by shuffles: (dp|ps) 0.92 vs
// 1.07 ms, (fs|ds) 0.67 vs 0.75 ms on the H100), picks the ket transfer of its own (k,l) powers, and runs the bra transfer,
// the root sum and the digestion for its own components only.  As in jk_tpq.cuh there is no shared memory and no barrier: the only cooperation
// inside a segment is that its lanes walk the same kets, so the screening decision and the primitive loops are uniform over it.
// A CTA owns one bra pair, J[ij] is accumulated in registers over all kets, reduced with warp shuffles and flushed once.
#pragma once
#include "jk_tpq.cuh"

namespace b200jk {

constexpr int SWQ_NACC = 36;   // accumulators per lane (the thread-per-quartet budget)

// lanes per quartet: the fewest of 2, 4, 8 that keep ceil(NKL / T) bra blocks within SWQ_NACC; 0 if none does
constexpr int swq_lanes(int nab, int nkl)
{
    for (int t = 2; t <= 8; t *= 2)
        if ((nkl + t - 1) / t * nab <= SWQ_NACC) return t;
    return 0;
}

// classes (as launched, bra | ket) that run on the sub-warp kernels: each is faster than its block kernel on the H100 by clearly
// more than the spread of repeated class timings (DESIGN.md §4.1).  (dp|pp) (T = 8, 9 of 16 lanes busy) and (fd|ss) (a 60-integral
// bra block, more than one lane can hold) stay on the block kernels.
constexpr bool swq_class(int li, int lj, int lk, int ll)
{
    return (li == 2 && lj == 1 && lk == 1 && ll == 0) ||   // (dp|ps)
           (li == 2 && lj == 0 && lk == 1 && ll == 1) ||   // (ds|pp)
           (li == 2 && lj == 1 && lk == 2 && ll == 0) ||   // (dp|ds)
           (li == 3 && lj == 0 && lk == 2 && ll == 0) ||   // (fs|ds)
           (li == 3 && lj == 1 && lk == 1 && ll == 0) ||   // (fp|ps)
           (li == 2 && lj == 2 && lk == 1 && ll == 0) ||   // (dd|ps)
           (li == 1 && lj == 1 && lk == 3 && ll == 0) ||   // (pp|fs), launched swapped
           (li == 1 && lj == 1 && lk == 1 && ll == 1);     // (pp|pp)
}

template <class C>
struct SwqCfg {
    static constexpr int NAB = C::NI * C::NJ, NKL = C::NKL;
    static constexpr int T = swq_lanes(NAB, NKL);       // lanes per quartet
    static constexpr int S = T ? (NKL + T - 1) / T : 1;  // ket component pairs per lane
    static constexpr bool eligible = swq_class(C::LI, C::LJ, C::LK, C::LL) && T > 0 && C::NR <= 3;
    static constexpr int NT = B2_TPQ_NT;                 // threads per CTA
    static constexpr int NSLOT = T ? NT / T : 1;         // quartet slots per CTA
    static constexpr int PSLICE = B2_TPQ_PSLICE;
    static constexpr int KCHUNK = B2_TPQ_KCHUNK;
    static constexpr int GI = C::LI + 1, GKL = (C::LK + 1) * (C::LL + 1);
};

// vertical recurrence of one direction and root, then the ket transfer (k -> l) for every (k,l):
// K[(l*(LK+1) + k)*NB1 + n], n = 0..LB the bra power before the bra transfer
template <class C>
B2_HD void swq_vrr(double c00, double c0p, double b00, double b10, double b01, double i00, double CD, double* K)
{
    double I[C::NB1][C::NT1];
    I[0][0] = i00;
    if (C::LB > 0) {
        I[1][0] = c00 * i00;
        B2_UNROLL
        for (int n = 1; n < C::LB; n++) I[n + 1][0] = c00 * I[n][0] + n * b10 * I[n - 1][0];
    }
    B2_UNROLL
    for (int m = 0; m < C::LT; m++) {
        B2_UNROLL
        for (int n = 0; n <= C::LB; n++) {
            double val = c0p * I[n][m];
            if (m > 0) val += m * b01 * I[n][m - 1];
            if (n > 0) val += n * b00 * I[n - 1][m];
            I[n][m + 1] = val;
        }
    }
    B2_UNROLL
    for (int l = 0; l <= C::LL; l++) {
        if (l > 0) {
            B2_UNROLL
            for (int n = 0; n <= C::LB; n++) {
                B2_UNROLL
                for (int m = 0; m <= C::LT - l; m++) I[n][m] = I[n][m + 1] + CD * I[n][m];
            }
        }
        B2_UNROLL
        for (int k = 0; k <= C::LK; k++) {
            B2_UNROLL
            for (int n = 0; n <= C::LB; n++) K[(l * (C::LK + 1) + k) * C::NB1 + n] = I[n][k];
        }
    }
}

// the row of the lane's ket powers (kl = l*(LK+1) + k, a run-time value) by selection, then the bra transfer (i -> j):
// g[j*(LI+1) + i]
template <class C>
B2_HD void swq_pick(const double* K, int kl, double AB, double* g)
{
    using W = SwqCfg<C>;
    double X[C::NB1];
    B2_UNROLL
    for (int n = 0; n <= C::LB; n++) X[n] = K[n];
    B2_UNROLL
    for (int e = 1; e < W::GKL; e++) {
        const bool m = (e == kl);
        B2_UNROLL
        for (int n = 0; n <= C::LB; n++) X[n] = m ? K[e * C::NB1 + n] : X[n];
    }
    B2_UNROLL
    for (int i = 0; i <= C::LI; i++) g[i] = X[i];
    B2_UNROLL
    for (int j = 1; j <= C::LJ; j++) {
        B2_UNROLL
        for (int n = 0; n <= C::LB - j; n++) X[n] = X[n + 1] + AB * X[n];
        B2_UNROLL
        for (int i = 0; i <= C::LI; i++) g[j * W::GI + i] = X[i];
    }
}

// the lane's ket components: kl index of the 2-D integral rows per direction
struct SwqLane {
    int kx[8], ky[8], kz[8];   // l*(LK+1) + k per direction, one entry per owned ket component pair (S <= 8)
};

// the lane's integrals of one shell quartet: v[s*NAB + b*NI + a] for ket component pair cd = t + s*T
template <class C, bool SR>
B2_HD void swq_eri(const KParams& P, const ShellPair& bp, const ShellPair& kp, int ib0, int ib1, const SwqLane& ln, double* v)
{
    using W = SwqCfg<C>;
    B2_UNROLL
    for (int e = 0; e < W::S * W::NAB; e++) v[e] = 0.0;
    for (int ik = 0; ik < kp.nprim; ik++) {
        const PrimPair k = load_prim(P.prims + kp.prim_off + ik);
        for (int ib = ib0; ib < ib1; ib++) {
            const PrimPair b = load_prim(P.prims + bp.prim_off + ib);
            double p = b.p, q = k.p;
            double PQx = b.Px - k.Px, PQy = b.Py - k.Py, PQz = b.Pz - k.Pz;
            double pq = p + q;
            double rs = rsqrt(pq);
            double ipq = rs * rs;
            double rho = p * q * ipq;
            double x = rho * (PQx * PQx + PQy * PQy + PQz * PQz);
            const double x0 = x, pref0 = b.cc * k.cc * rs;
            double hip = 0.5 / p, hiq = 0.5 / q;
            if (C::LB == 0) hip = 0.0;
            if (C::LT == 0) hiq = 0.0;
            // omega < 0 (erfc = Coulomb - erf): a second pass over the roots with the erf-attenuated set, weights negated
            constexpr int nsr = SR ? 2 : 1;
            B2_NOUNROLL
            for (int sr = 0; sr < nsr; sr++) {
            double pref = pref0;
            double theta = 1.0;
            const double om = (nsr == 2) ? (sr ? -P.omega : 0.0) : P.omega;
            x = x0;
            if (om > 0.0) {
                theta = om * om / (om * om + rho);
                x *= theta;
                pref *= sqrt(theta);
            }
            if (sr) pref = -pref;
            B2_NOUNROLL
            for (int r = 0; r < C::NR; r++) {
                double u, w;
                rys_root(P.tb, C::NR, r, x, u, w);
                u *= theta; w *= pref;
                double b00 = 0.5 * u * ipq;
                double b10 = (1.0 - u * q * ipq) * hip;
                double b01 = (1.0 - u * p * ipq) * hiq;
                double uq = u * q * ipq, up = u * p * ipq;
                double Kx[W::GKL * C::NB1], Ky[W::GKL * C::NB1], Kz[W::GKL * C::NB1];
                swq_vrr<C>(b.PAx - uq * PQx, k.PAx + up * PQx, b00, b10, b01, 1.0, kp.ABx, Kx);
                swq_vrr<C>(b.PAy - uq * PQy, k.PAy + up * PQy, b00, b10, b01, 1.0, kp.ABy, Ky);
                swq_vrr<C>(b.PAz - uq * PQz, k.PAz + up * PQz, b00, b10, b01, w, kp.ABz, Kz);
                B2_UNROLL
                for (int s = 0; s < W::S; s++) {
                    double gx[W::GI * (C::LJ + 1)], gy[W::GI * (C::LJ + 1)], gz[W::GI * (C::LJ + 1)];
                    swq_pick<C>(Kx, ln.kx[s], bp.ABx, gx);
                    swq_pick<C>(Ky, ln.ky[s], bp.ABy, gy);
                    swq_pick<C>(Kz, ln.kz[s], bp.ABz, gz);
                    B2_UNROLL
                    for (int bb = 0; bb < C::NJ; bb++) {
                        B2_UNROLL
                        for (int a = 0; a < C::NI; a++) {
                            const int ix = cart_px(C::LI, a), iy = cart_py(C::LI, a), iz = C::LI - ix - iy;
                            const int jx = cart_px(C::LJ, bb), jy = cart_py(C::LJ, bb), jz = C::LJ - jx - jy;
                            v[s * W::NAB + bb * C::NI + a] +=
                                gx[jx * W::GI + ix] * gy[jy * W::GI + iy] * gz[jz * W::GI + iz];
                        }
                    }
                }
            }
            }
        }
    }
}

// digestion of the lane's bra block for ONE ket component pair (kc, ld) (the update rules of phase_digest)
// one_j (n_dm_j == 1): J[ij] of the stationary bra pair goes to the registers jij, flushed once per CTA.  D[ij] is read
// through L1 rather than held in registers: next to the accumulators and jij it would push the kernels into spills.
template <class C>
B2_HD void swq_digest(const KParams& P, const double* v, double f, int i0, int j0, int kc, int ld, bool one_j, double* jij)
{
    using W = SwqCfg<C>;
    const int n = P.n;
    const size_t n2 = (size_t)n * n;
    if (P.vj) {
        for (int idm = 0; idm < P.n_dm_j; idm++) {
            const double* D = P.dmj + idm * n2;
            double* J = P.vj + idm * n2;
            const double dkl = 2.0 * f * B2_LDG(&D[(size_t)kc * n + ld]);
            double jkl = 0.0;
            B2_UNROLL
            for (int e = 0; e < W::NAB; e++) {
                const size_t ij = (size_t)(i0 + e % C::NI) * n + j0 + e / C::NI;
                jkl += v[e] * B2_LDG(&D[ij]);
                if (one_j) jij[e] += v[e] * dkl;
                else red_add(&J[ij], v[e] * dkl);
            }
            red_add(&J[(size_t)kc * n + ld], 2.0 * f * jkl);
        }
    }
    if (P.vk) {
        for (int idm = 0; idm < P.n_dm_k; idm++) {
            const double* D = P.dmk + idm * n2;
            double* K = P.vk + idm * n2;
            double kik[C::NI], kil[C::NI], dik[C::NI], dil[C::NI], kjk[C::NJ], kjl[C::NJ], djk[C::NJ], djl[C::NJ];
            B2_UNROLL
            for (int a = 0; a < C::NI; a++) {
                kik[a] = 0.0; kil[a] = 0.0;
                dik[a] = B2_LDG(&D[(size_t)(i0 + a) * n + kc]);
                dil[a] = B2_LDG(&D[(size_t)(i0 + a) * n + ld]);
            }
            B2_UNROLL
            for (int bb = 0; bb < C::NJ; bb++) {
                djk[bb] = B2_LDG(&D[(size_t)(j0 + bb) * n + kc]);
                djl[bb] = B2_LDG(&D[(size_t)(j0 + bb) * n + ld]);
            }
            B2_UNROLL
            for (int bb = 0; bb < C::NJ; bb++) {
                double sjk = 0.0, sjl = 0.0;
                B2_UNROLL
                for (int a = 0; a < C::NI; a++) {
                    const double val = v[bb * C::NI + a];
                    kik[a] += val * djl[bb];
                    kil[a] += val * djk[bb];
                    sjk += val * dil[a];
                    sjl += val * dik[a];
                }
                kjk[bb] = sjk; kjl[bb] = sjl;
            }
            B2_UNROLL
            for (int a = 0; a < C::NI; a++) {
                red_add(&K[(size_t)(i0 + a) * n + kc], f * kik[a]);
                red_add(&K[(size_t)(i0 + a) * n + ld], f * kil[a]);
            }
            B2_UNROLL
            for (int bb = 0; bb < C::NJ; bb++) {
                red_add(&K[(size_t)(j0 + bb) * n + kc], f * kjk[bb]);
                red_add(&K[(size_t)(j0 + bb) * n + ld], f * kjl[bb]);
            }
        }
    }
}

template <class C, bool SR>
#ifdef __CUDACC__
__device__ __forceinline__
#else
inline
#endif
void swq_block(const KParams& P, int bx, int by, int bz)
{
    using W = SwqCfg<C>;
    static_assert(W::T > 0 && W::S <= 8 && 32 % W::T == 0, "sub-warp layout");
    const ShellPair bpair = P.bra_pairs[bx];
    const int kmax = P.same_class ? (bx + 1) : P.nket;
    const int kbeg = by * P.kchunk;
    const int kend = (kbeg + P.kchunk < kmax) ? kbeg + P.kchunk : kmax;
    if (kbeg >= kend) return;
    const int ib0 = bz * P.pslice;
    const int ib1 = (ib0 + P.pslice < bpair.nprim) ? ib0 + P.pslice : bpair.nprim;
    if (ib0 >= ib1) return;
#if defined(__CUDA_ARCH__)
    {
        const int tid = threadIdx.x;
#else
    double jsum[W::NAB];
    for (int e = 0; e < W::NAB; e++) jsum[e] = 0.0;
    unsigned long long ncomp = 0, nskip = 0;
    for (int tid = 0; tid < W::NT; tid++) {
#endif
        const int slot = tid / W::T, t = tid % W::T;
        SwqLane ln;
        int cof[W::S], dof[W::S];
        B2_UNROLL
        for (int s = 0; s < W::S; s++) {
            int cd = t + s * W::T;
            if (cd >= W::NKL) cd = 0;   // idle slot: computed, never digested
            const int c = cd % C::NK, d = cd / C::NK;
            cof[s] = c; dof[s] = d;
            ln.kx[s] = cart_px(C::LL, d) * (C::LK + 1) + cart_px(C::LK, c);
            ln.ky[s] = cart_py(C::LL, d) * (C::LK + 1) + cart_py(C::LK, c);
            ln.kz[s] = cart_pz(C::LL, d) * (C::LK + 1) + cart_pz(C::LK, c);
        }
        double jij[W::NAB];
        const bool one_j = P.vj && P.n_dm_j == 1;
        B2_UNROLL
        for (int e = 0; e < W::NAB; e++) jij[e] = 0.0;
        int mine = 0, skipped = 0;
        for (int kk = kbeg + slot; kk < kend; kk += W::NSLOT) {
            const ShellPair kp = load_pair(P.ket_pairs + kk);
            if (!keep_quartet(bpair.q, kp.q, bpair.ish, bpair.jsh, kp.ish, kp.jsh, P.dmc, P.nsh, P.tol, P.vj != nullptr,
                              P.vk != nullptr)) {
                if (bz == 0 && t == 0) skipped++;
                continue;
            }
            if (bz == 0 && t == 0) mine++;
            double f = 1.0;
            if (bpair.same) f *= 0.5;
            if (kp.same) f *= 0.5;
            if (P.same_class && kk == bx) f *= 0.5;
            double v[W::S * W::NAB];
            swq_eri<C, SR>(P, bpair, kp, ib0, ib1, ln, v);
            B2_UNROLL
            for (int s = 0; s < W::S; s++)
                if (t + s * W::T < W::NKL)
                    swq_digest<C>(P, v + s * W::NAB, f, bpair.i0, bpair.j0, kp.i0 + cof[s], kp.j0 + dof[s], one_j, jij);
        }
#if defined(__CUDA_ARCH__)
        // warp-reduce the stationary J[ij] block, one reduction per warp and element
        if (one_j) {
            B2_UNROLL
            for (int e = 0; e < W::NAB; e++) {
                double val = jij[e];
                B2_UNROLL
                for (int o = 16; o > 0; o >>= 1) val += __shfl_xor_sync(0xffffffffu, val, o);
                if ((tid & 31) == 0 && val != 0.0)
                    atomicAdd(&P.vj[(size_t)(bpair.i0 + e % C::NI) * P.n + bpair.j0 + e / C::NI], val);
            }
        }
        if (P.counters) {
            int tot = mine;
            B2_UNROLL
            for (int o = 16; o > 0; o >>= 1) tot += __shfl_xor_sync(0xffffffffu, tot, o);
            int sk = skipped;
            B2_UNROLL
            for (int o = 16; o > 0; o >>= 1) sk += __shfl_xor_sync(0xffffffffu, sk, o);
            if ((tid & 31) == 0) {
                atomicAdd(&P.counters[0], (unsigned long long)tot);
                atomicAdd(&P.counters[1], (unsigned long long)sk);
            }
        }
    }
#else
        for (int e = 0; e < W::NAB; e++) jsum[e] += jij[e];
        ncomp += mine;
        nskip += skipped;
    }
    if (P.vj && P.n_dm_j == 1)
        for (int e = 0; e < W::NAB; e++) P.vj[(size_t)(bpair.i0 + e % C::NI) * P.n + bpair.j0 + e / C::NI] += jsum[e];
    if (P.counters) { P.counters[0] += ncomp; P.counters[1] += nskip; }
#endif
}

}  // namespace b200jk
