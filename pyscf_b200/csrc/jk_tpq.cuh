// jk_tpq.cuh — "thread per quartet" kernels for the low angular-momentum classes
// ((ab|cd) blocks of <= 36 Cartesian integrals, nroots <= 3): ss|ss ... ds|ds, dd|ss, fs|ps, fp|ss.
//
// These classes carry the deeply contracted s/p shells (most primitive quartets) but almost no
// arithmetic per primitive, so the cooperative shared-memory pipeline of jk_block.cuh is dominated by
// synchronisation.  Here one thread owns a whole shell quartet: Rys roots, both recurrences, the root
// sum and the digestion all stay in registers; there is no shared memory and no barrier.  A CTA still
// owns one bra pair, so J[ij] is accumulated in registers over all kets, reduced with warp shuffles
// and flushed once.
#pragma once
#include "jk_block.cuh"

namespace b200jk {

// compile-time tuning knobs of the thread-per-quartet kernels (A/B libraries: tools/build_variant.sh)
#ifndef B2_TPQ_NT
#define B2_TPQ_NT 128        // threads per CTA
#endif
#ifndef B2_TPQ_PSLICE
#define B2_TPQ_PSLICE 8      // bra primitive pairs per CTA slice
#endif
#ifndef B2_TPQ_KOUTER
#define B2_TPQ_KOUTER 1      // 1: ket primitive loop outside the bra primitive loop (each thread loads its own ket primitive once
#endif                       //    per ket primitive instead of once per primitive QUARTET; the bra primitive is warp-uniform).
                             //    Chosen by A/B timing on an earlier GPU generation; not re-measured on the H100.
#ifndef B2_TPQ_KCHUNK
#define B2_TPQ_KCHUNK 512    // ket pairs examined per CTA (upper bound)
#endif

template <class C>
struct TpqCfg {
    static constexpr int NAB = C::NI * C::NJ, NKL = C::NKL, NOUT = NAB * NKL;
    static constexpr bool eligible = (NOUT <= 36) && (C::NR <= 3) && (C::NP == 1);
    static constexpr int NT = B2_TPQ_NT;
    static constexpr int KCHUNK = B2_TPQ_KCHUNK;
    static constexpr int PSLICE = B2_TPQ_PSLICE;      // bra primitive pairs per CTA slice (blockIdx.z): bounds the serial work of a thread
    static constexpr int GI = C::LI + 1, GJ = C::LJ + 1, GK = C::LK + 1, GL = C::LL + 1;
    static constexpr int GSZ = GI * GJ * GK * GL;
};

// 2-D integrals of one direction for one root, all four indices, in registers:
// G[((l*GK + k)*GJ + j)*GI + i]
template <class C>
B2_HD void tpq_g2d(double c00, double c0p, double b00, double b10, double b01, double i00, double AB, double CD, double* G)
{
    using T = TpqCfg<C>;
    constexpr int NB1 = C::NB1, NT1 = C::NT1;
    double I[NB1][NT1];
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
    // ket transfer (k -> l) level by level, then bra transfer (i -> j) for every (k,l)
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
            double X[NB1];
            B2_UNROLL
            for (int n = 0; n <= C::LB; n++) X[n] = I[n][k];
            B2_UNROLL
            for (int i = 0; i <= C::LI; i++) G[((l * T::GK + k) * T::GJ + 0) * T::GI + i] = X[i];
            B2_UNROLL
            for (int j = 1; j <= C::LJ; j++) {
                B2_UNROLL
                for (int n = 0; n <= C::LB - j; n++) X[n] = X[n + 1] + AB * X[n];
                B2_UNROLL
                for (int i = 0; i <= C::LI; i++) G[((l * T::GK + k) * T::GJ + j) * T::GI + i] = X[i];
            }
        }
    }
}

// all Cartesian integrals of one shell quartet: v[(d*NK + c)*NAB + b*NI + a]
template <class C, bool SR>
B2_HD void tpq_eri(const KParams& P, const ShellPair& bp, const ShellPair& kp, int ib0, int ib1, double* v)
{
    using T = TpqCfg<C>;
    B2_UNROLL
    for (int e = 0; e < T::NOUT; e++) v[e] = 0.0;
#if B2_TPQ_KOUTER
    for (int ik = 0; ik < kp.nprim; ik++) {
        const PrimPair k = load_prim(P.prims + kp.prim_off + ik);
        for (int ib = ib0; ib < ib1; ib++) {
            const PrimPair b = load_prim(P.prims + bp.prim_off + ib);
#else
    for (int ib = ib0; ib < ib1; ib++) {
        const PrimPair b = load_prim(P.prims + bp.prim_off + ib);
        for (int ik = 0; ik < kp.nprim; ik++) {
            const PrimPair k = load_prim(P.prims + kp.prim_off + ik);
#endif
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
            B2_UNROLL
            for (int r = 0; r < C::NR; r++) {
                double u, w;
                rys_root(P.tb, C::NR, r, x, u, w);
                u *= theta; w *= pref;
                double b00 = 0.5 * u * ipq;
                double b10 = (1.0 - u * q * ipq) * hip;
                double b01 = (1.0 - u * p * ipq) * hiq;
                double uq = u * q * ipq, up = u * p * ipq;
                double Gx[T::GSZ], Gy[T::GSZ], Gz[T::GSZ];
                tpq_g2d<C>(b.PAx - uq * PQx, k.PAx + up * PQx, b00, b10, b01, 1.0, bp.ABx, kp.ABx, Gx);
                tpq_g2d<C>(b.PAy - uq * PQy, k.PAy + up * PQy, b00, b10, b01, 1.0, bp.ABy, kp.ABy, Gy);
                tpq_g2d<C>(b.PAz - uq * PQz, k.PAz + up * PQz, b00, b10, b01, w, bp.ABz, kp.ABz, Gz);
                B2_UNROLL
                for (int d = 0; d < C::NL; d++) {
                    B2_UNROLL
                    for (int c = 0; c < C::NK; c++) {
                        B2_UNROLL
                        for (int bb = 0; bb < C::NJ; bb++) {
                            B2_UNROLL
                            for (int a = 0; a < C::NI; a++) {
                                const int ix = cart_px(C::LI, a), iy = cart_py(C::LI, a), iz = C::LI - ix - iy;
                                const int jx = cart_px(C::LJ, bb), jy = cart_py(C::LJ, bb), jz = C::LJ - jx - jy;
                                const int kx = cart_px(C::LK, c), ky = cart_py(C::LK, c), kz = C::LK - kx - ky;
                                const int lx = cart_px(C::LL, d), ly = cart_py(C::LL, d), lz = C::LL - lx - ly;
                                v[(d * C::NK + c) * T::NAB + bb * C::NI + a] +=
                                    Gx[((lx * T::GK + kx) * T::GJ + jx) * T::GI + ix] *
                                    Gy[((ly * T::GK + ky) * T::GJ + jy) * T::GI + iy] *
                                    Gz[((lz * T::GK + kz) * T::GJ + jz) * T::GI + iz];
                            }
                        }
                    }
                }
            }
            }
        }
    }
}

// digestion of one quartet held entirely by one thread (same update rules as phase_digest)
// dij_pre: the D[ij] block of the stationary bra pair, loaded once per thread (n_dm_j == 1), else nullptr.
// All density elements are fetched BEFORE the first reduction is issued: a load placed after a RED cannot be hoisted
// above it (possible alias), which would serialise every (c,d) step on the load latency and re-read D[ij] each time.
template <class C>
B2_HD void tpq_digest(const KParams& P, const double* v, double f, int i0, int j0, int k0, int l0, double* jij, const double* dij_pre)
{
    using T = TpqCfg<C>;
    const int n = P.n;
    const size_t n2 = (size_t)n * n;
    if (P.vj) {
        for (int idm = 0; idm < P.n_dm_j; idm++) {
            const double* D = P.dmj + idm * n2;
            double* J = P.vj + idm * n2;
            double jab[T::NAB], dij[T::NAB], dkl[C::NK * C::NL], jkl[C::NK * C::NL];
            B2_UNROLL
            for (int e = 0; e < C::NK * C::NL; e++) dkl[e] = B2_LDG(&D[(size_t)(k0 + e % C::NK) * n + l0 + e / C::NK]);
            B2_UNROLL
            for (int e = 0; e < T::NAB; e++) {
                jab[e] = 0.0;
                dij[e] = dij_pre ? dij_pre[e] : B2_LDG(&D[(size_t)(i0 + e % C::NI) * n + j0 + e / C::NI]);
            }
            B2_UNROLL
            for (int d = 0; d < C::NL; d++) {
                B2_UNROLL
                for (int c = 0; c < C::NK; c++) {
                    double acc = 0.0;
                    B2_UNROLL
                    for (int e = 0; e < T::NAB; e++) {
                        double val = v[(d * C::NK + c) * T::NAB + e];
                        acc += val * dij[e];
                        jab[e] += val * dkl[d * C::NK + c];
                    }
                    jkl[d * C::NK + c] = acc;
                }
            }
            B2_UNROLL
            for (int e = 0; e < C::NK * C::NL; e++) red_add(&J[(size_t)(k0 + e % C::NK) * n + l0 + e / C::NK], 2.0 * f * jkl[e]);
            if (P.n_dm_j == 1) {
                B2_UNROLL
                for (int e = 0; e < T::NAB; e++) jij[e] += 2.0 * f * jab[e];
            } else {
                B2_UNROLL
                for (int bb = 0; bb < C::NJ; bb++) {
                    B2_UNROLL
                    for (int a = 0; a < C::NI; a++) red_add(&J[(size_t)(i0 + a) * n + j0 + bb], 2.0 * f * jab[bb * C::NI + a]);
                }
            }
        }
    }
    if (P.vk) {
        for (int idm = 0; idm < P.n_dm_k; idm++) {
            const double* D = P.dmk + idm * n2;
            double* K = P.vk + idm * n2;
            double kik[C::NI * C::NK], kil[C::NI * C::NL], kjk[C::NJ * C::NK], kjl[C::NJ * C::NL];
            B2_UNROLL
            for (int e = 0; e < C::NI * C::NK; e++) kik[e] = 0.0;
            B2_UNROLL
            for (int e = 0; e < C::NI * C::NL; e++) kil[e] = 0.0;
            B2_UNROLL
            for (int e = 0; e < C::NJ * C::NK; e++) kjk[e] = 0.0;
            B2_UNROLL
            for (int e = 0; e < C::NJ * C::NL; e++) kjl[e] = 0.0;
            B2_UNROLL
            for (int d = 0; d < C::NL; d++) {
                B2_UNROLL
                for (int c = 0; c < C::NK; c++) {
                    B2_UNROLL
                    for (int bb = 0; bb < C::NJ; bb++) {
                        double djl = B2_LDG(&D[(size_t)(j0 + bb) * n + l0 + d]), djk = B2_LDG(&D[(size_t)(j0 + bb) * n + k0 + c]);
                        B2_UNROLL
                        for (int a = 0; a < C::NI; a++) {
                            double val = v[(d * C::NK + c) * T::NAB + bb * C::NI + a];
                            double dil = B2_LDG(&D[(size_t)(i0 + a) * n + l0 + d]), dik = B2_LDG(&D[(size_t)(i0 + a) * n + k0 + c]);
                            kik[a * C::NK + c] += val * djl;
                            kil[a * C::NL + d] += val * djk;
                            kjk[bb * C::NK + c] += val * dil;
                            kjl[bb * C::NL + d] += val * dik;
                        }
                    }
                }
            }
            B2_UNROLL
            for (int a = 0; a < C::NI; a++) {
                B2_UNROLL
                for (int c = 0; c < C::NK; c++) red_add(&K[(size_t)(i0 + a) * n + k0 + c], f * kik[a * C::NK + c]);
                B2_UNROLL
                for (int d = 0; d < C::NL; d++) red_add(&K[(size_t)(i0 + a) * n + l0 + d], f * kil[a * C::NL + d]);
            }
            B2_UNROLL
            for (int bb = 0; bb < C::NJ; bb++) {
                B2_UNROLL
                for (int c = 0; c < C::NK; c++) red_add(&K[(size_t)(j0 + bb) * n + k0 + c], f * kjk[bb * C::NK + c]);
                B2_UNROLL
                for (int d = 0; d < C::NL; d++) red_add(&K[(size_t)(j0 + bb) * n + l0 + d], f * kjl[bb * C::NL + d]);
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
void tpq_block(const KParams& P, int bx, int by, int bz)
{
    using T = TpqCfg<C>;
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
    double jsum[T::NAB];
    for (int e = 0; e < T::NAB; e++) jsum[e] = 0.0;
    unsigned long long ncomp = 0, nskip = 0;
    for (int tid = 0; tid < T::NT; tid++) {
#endif
        double jij[T::NAB], dij[T::NAB];
        const bool one_j = P.vj && P.n_dm_j == 1;
        B2_UNROLL
        for (int e = 0; e < T::NAB; e++) {
            jij[e] = 0.0;
            dij[e] = one_j ? B2_LDG(&P.dmj[(size_t)(bpair.i0 + e % C::NI) * P.n + bpair.j0 + e / C::NI]) : 0.0;
        }
        int mine = 0, skipped = 0;
        for (int kk = kbeg + tid; kk < kend; kk += T::NT) {
            const ShellPair kp = load_pair(P.ket_pairs + kk);
            if (!keep_quartet(bpair.q, kp.q, bpair.ish, bpair.jsh, kp.ish, kp.jsh, P.dmc, P.nsh, P.tol, P.vj != nullptr,
                              P.vk != nullptr)) {
                if (bz == 0) skipped++;
                continue;
            }
            if (bz == 0) mine++;
            double f = 1.0;
            if (bpair.same) f *= 0.5;
            if (kp.same) f *= 0.5;
            if (P.same_class && kk == bx) f *= 0.5;
            double v[T::NOUT];
            tpq_eri<C, SR>(P, bpair, kp, ib0, ib1, v);
            tpq_digest<C>(P, v, f, bpair.i0, bpair.j0, kp.i0, kp.j0, jij, one_j ? dij : nullptr);
        }
#if defined(__CUDA_ARCH__)
        // warp-reduce the stationary J[ij] block, one reduction per warp and element
        if (P.vj && P.n_dm_j == 1) {
            B2_UNROLL
            for (int e = 0; e < T::NAB; e++) {
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
        for (int e = 0; e < T::NAB; e++) jsum[e] += jij[e];
        ncomp += mine;
        nskip += skipped;
    }
    if (P.vj && P.n_dm_j == 1)
        for (int e = 0; e < T::NAB; e++) P.vj[(size_t)(bpair.i0 + e % C::NI) * P.n + bpair.j0 + e / C::NI] += jsum[e];
    if (P.counters) { P.counters[0] += ncomp; P.counters[1] += nskip; }
#endif
}

}  // namespace b200jk
