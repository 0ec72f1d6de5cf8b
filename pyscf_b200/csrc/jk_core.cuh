// jk_core.cuh — device-side arithmetic of the 4-center direct J/K path (sm_90a), written so that
// the same templates also compile with g++ for the CPU SIMT-emulation tests (tests/emu).
//
// Replaces (reference file:line):
//   libcint int2e_sph (Rys quadrature)       called at pyscf/lib/vhf/nr_direct.c:73
//   nrs8_ji_s2kl / nrs8_li_s2kj digestion    pyscf/lib/vhf/nr_direct_dot.c:1293,1435
//   CVHFnrs8_prescreen                       pyscf/lib/vhf/optimizer.c:90-117
// Design (DESIGN.md §3): one kernel per angular-momentum class (LI LJ|LK LL).  A CTA owns one bra
// shell pair (ij) and walks a screened list of ket pairs (kl), NQ at a time.  Inside a quartet the
// ket Cartesian component pair (c,d) is the THREAD index and the bra component block (a,b) lives in
// REGISTERS; the 2-D Rys integrals I(n,m) are produced cooperatively into shared memory and each
// thread applies the horizontal recurrences for its own (c,d) in registers.  ERIs are never
// stored: they are contracted with the density in registers and flushed as fp64 reductions.
#pragma once
#include <math.h>
#include <stdint.h>

#ifdef __CUDACC__
#define B2_HD __host__ __device__ __forceinline__
#define B2_UNROLL _Pragma("unroll")
#define B2_NOUNROLL _Pragma("unroll 1")
#else
#define B2_HD inline __attribute__((always_inline))
#define B2_UNROLL
#define B2_NOUNROLL
#endif

namespace b200jk {

#ifndef __CUDACC__
inline double rsqrt(double x) { return 1.0 / sqrt(x); }
#endif

constexpr int LMAX = 4;  // g shells (aux); orbital classes are generated up to f
constexpr int RYS_NMAX = 9, RYS_DEG = 7, RYS_NINT = 320;   // degree-7 Chebyshev pieces on 320 intervals of 0.3125
constexpr double RYS_H = 0.3125, RYS_XMAX = 100.0;
constexpr int RYS_ROW = 2 * (RYS_DEG + 1);                  // doubles per (interval, root): node and weight polynomials
constexpr double PI_25_2 = 34.98683665524972497;  // 2*pi^(5/2)

B2_HD constexpr int ncart(int l) { return (l + 1) * (l + 2) / 2; }

// libcint Cartesian order: lx descending, then ly descending (pyscf/lib/parameters.py:69-77)
B2_HD constexpr int cart_px(int l, int a)
{
    int n = 0;
    for (int x = l; x >= 0; x--)
        for (int y = l - x; y >= 0; y--) {
            if (n == a) return x;
            n++;
        }
    return 0;
}
B2_HD constexpr int cart_py(int l, int a)
{
    int n = 0;
    for (int x = l; x >= 0; x--)
        for (int y = l - x; y >= 0; y--) {
            if (n == a) return y;
            n++;
        }
    return 0;
}
B2_HD constexpr int cart_pz(int l, int a) { return l - cart_px(l, a) - cart_py(l, a); }

// ---------------------------------------------------------------------------------------------
// Rys roots and weights from the tables made by tools/gen_rys_tables.py
struct RysTables {
    const double* herm;  // for n: offset n(n-1): u_r*x (n values), w_r*sqrt(x) (n values)
    const double* cheb;  // for n: offset NINT*RYS_ROW*n(n-1)/2: [NINT][n][2][DEG+1]
};

B2_HD void rys_root(const RysTables& tb, int n, int r, double x, double& u, double& w)
{
    if (x >= RYS_XMAX) {
        const double* h = tb.herm + n * (n - 1);
        double ix = 1.0 / x;
        u = h[r] * ix;
        w = h[n + r] * sqrt(ix);
        return;
    }
    int iv = (int)(x * (1.0 / RYS_H));
    if (iv > RYS_NINT - 1) iv = RYS_NINT - 1;
    double t = (x - iv * RYS_H) * (2.0 / RYS_H) - 1.0;
    const double* cp = tb.cheb + (size_t)RYS_NINT * RYS_ROW * (n * (n - 1) / 2) + (size_t)(iv * n + r) * RYS_ROW;
    double c[RYS_ROW];
#if defined(__CUDA_ARCH__)
    // one table row = 128 B = 8 x 128-bit loads (the widest global load of sm_90); rows are 32-byte aligned (b200jk_create)
    B2_UNROLL
    for (int j = 0; j < RYS_ROW / 2; j++)
        asm volatile("ld.global.nc.v2.f64 {%0,%1}, [%2];" : "=d"(c[2 * j]), "=d"(c[2 * j + 1]) : "l"(cp + 2 * j));
#else
    for (int j = 0; j < RYS_ROW; j++) c[j] = cp[j];
#endif
    double t2 = 2.0 * t, b1 = 0.0, b2 = 0.0, d1 = 0.0, d2 = 0.0;
    B2_UNROLL
    for (int j = RYS_DEG; j >= 1; j--) {
        double tb_ = t2 * b1 - b2 + c[j];
        b2 = b1; b1 = tb_;
        double td_ = t2 * d1 - d2 + c[RYS_DEG + 1 + j];
        d2 = d1; d1 = td_;
    }
    u = t * b1 - b2 + c[0];
    w = t * d1 - d2 + c[RYS_DEG + 1];
}

// ---------------------------------------------------------------------------------------------
// Shell-pair data (HBM layout, DESIGN.md §2)
struct PrimPair {  // 64 bytes, one per surviving primitive pair
    double p;             // a_i + a_j
    double Px, Py, Pz;    // Gaussian product centre
    double PAx, PAy, PAz; // P - A   (A = centre of the first shell of the pair)
    double cc;            // sqrt(2 pi^(5/2)) * c_i c_j exp(-a_i a_j |AB|^2 / p) / p
};
// one PrimPair = 64 B = four 128-bit loads (half the L1 tag traffic of eight 64-bit loads)
B2_HD PrimPair load_prim(const PrimPair* p)
{
#if defined(__CUDA_ARCH__)
    PrimPair r;
    const double* d = (const double*)p;
    asm volatile("ld.global.nc.v2.f64 {%0,%1}, [%2];" : "=d"(r.p), "=d"(r.Px) : "l"(d));
    asm volatile("ld.global.nc.v2.f64 {%0,%1}, [%2];" : "=d"(r.Py), "=d"(r.Pz) : "l"(d + 2));
    asm volatile("ld.global.nc.v2.f64 {%0,%1}, [%2];" : "=d"(r.PAx), "=d"(r.PAy) : "l"(d + 4));
    asm volatile("ld.global.nc.v2.f64 {%0,%1}, [%2];" : "=d"(r.PAz), "=d"(r.cc) : "l"(d + 6));
    return r;
#else
    return *p;
#endif
}

struct ShellPair {  // 64 bytes
    double ABx, ABy, ABz;  // A - B
    double q;              // Schwarz bound sqrt(max |(ab|ab)|) over Cartesian components
    int32_t ish, jsh;      // device shell ids
    int32_t i0, j0;        // Cartesian AO offsets
    int32_t prim_off, nprim;
    int32_t same;          // ish == jsh
    int32_t pad;
};

static_assert(sizeof(ShellPair) == 64, "ShellPair is loaded as four 128-bit words");
// one ShellPair = 64 B = four 128-bit loads
B2_HD ShellPair load_pair(const ShellPair* p)
{
#if defined(__CUDA_ARCH__)
    ShellPair r;
    unsigned long long w0, w1, w2, w3;
    const double* d = (const double*)p;
    asm volatile("ld.global.nc.v2.f64 {%0,%1}, [%2];" : "=d"(r.ABx), "=d"(r.ABy) : "l"(d));
    asm volatile("ld.global.nc.v2.f64 {%0,%1}, [%2];" : "=d"(r.ABz), "=d"(r.q) : "l"(d + 2));
    asm volatile("ld.global.nc.v2.u64 {%0,%1}, [%2];" : "=l"(w0), "=l"(w1) : "l"(d + 4));
    asm volatile("ld.global.nc.v2.u64 {%0,%1}, [%2];" : "=l"(w2), "=l"(w3) : "l"(d + 6));
    r.ish = (int32_t)(w0 & 0xffffffffu); r.jsh = (int32_t)(w0 >> 32);
    r.i0 = (int32_t)(w1 & 0xffffffffu); r.j0 = (int32_t)(w1 >> 32);
    r.prim_off = (int32_t)(w2 & 0xffffffffu); r.nprim = (int32_t)(w2 >> 32);
    r.same = (int32_t)(w3 & 0xffffffffu); r.pad = 0;
    return r;
#else
    return *p;
#endif
}

constexpr int MAX_PRIM_PER_PAIR = 16;   // pair lists are split so that no entry carries more primitive pairs (b200jk.cu)

// ---------------------------------------------------------------------------------------------
// PB_: primitive quartets processed per phase round by the block kernels (primitive batching): the Rys roots and the
// vertical recurrences of PB_ primitive quartets are spread over the lanes of a group TOGETHER, so that groups with many
// lanes (high angular momentum kets) are not idle while a handful of (root, direction) tasks run.  1 = one at a time.
template <int LI_, int LJ_, int LK_, int LL_, int NP_, int PB_ = 1>
struct QClass {
    static constexpr int LI = LI_, LJ = LJ_, LK = LK_, LL = LL_, NP = NP_, PB = PB_;
    static constexpr int NI = ncart(LI), NJ = ncart(LJ), NK = ncart(LK), NL = ncart(LL);
    static_assert(NJ % NP == 0, "NP must divide the number of j components");
    static constexpr int NJP = NJ / NP;
    static constexpr int NV = NI * NJP;   // register accumulators per thread
    static constexpr int NKL = NK * NL;
    static constexpr int G = NKL * NP;    // threads per quartet
    static constexpr int NR = (LI + LJ + LK + LL) / 2 + 1;
    static constexpr int LB = LI + LJ, LT = LK + LL, NB1 = LB + 1, NT1 = LT + 1, ISZ = NB1 * NT1;
    static constexpr int NI1 = LI + 1, NJ1 = LJ + 1;
    static constexpr int GK = (LK + 1) * (LL + 1);      // ket (k,l) index pairs of the 2-D integrals
    static constexpr int NB1P = (NB1 + 1) & ~1;           // bra length padded to an even count (16-byte rows)
    static constexpr int HSZ = GK * NB1P;
    static constexpr int HSP = HSZ + 2;                   // stride of one (direction, root) array: keeps 16-byte alignment
};

template <class C>
struct alignas(16) SlotSmem {
    // 2-D integrals after the vertical recurrence AND the ket transfer (k -> l), ready for per-thread bra transfer:
    // H[dir][root][(l*(LK+1)+k)*NB1P + n]; z carries weight*prefactor.  Rows of n are contiguous (LDS.128).
    // The leading index is the primitive quartet of the current batch (C::PB of them, see QClass).
    // The ket's primitive pairs are not staged here: phase A reads the one it needs from global memory (load_prim), so a
    // slot costs shared memory only for what phases B and D share between lanes.
    double H[C::PB][3][C::NR][C::HSP];
    double U[C::PB][C::NR], W[C::PB][C::NR];
    double pc[C::PB][14];        // p, q, PA[3], QC[3], PQ[3], 1/(p+q), 0.5/p, 0.5/q
    double ccd[3][C::LL + 1][C::LL + 1];  // binom(l,t) CD^(l-t)
    double fac;                  // symmetry factor (1, 1/2, 1/4, 1/8)
    int32_t kl, k0, l0, nprim_k, prim_off_k, active, pact, nq;   // nq: primitive quartets of this (bra, ket) (batched path)
};

struct BraInfo {
    double ABx, ABy, ABz;
    int32_t i0, j0, nprim, prim_off, same, idx;
};

template <class C>
struct ThreadCtx {
    int q, g, p, c, d;
    int kx, ky, kz, lx, ly, lz;
    double v[C::NV];
};

template <class C>
B2_HD void thread_decode(ThreadCtx<C>& t, int tid)
{
    t.q = tid / C::G;
    t.g = tid % C::G;
    t.p = t.g / C::NKL;
    int cd = t.g % C::NKL;
    t.c = cd % C::NK;
    t.d = cd / C::NK;
    t.kx = cart_px(C::LK, t.c); t.ky = cart_py(C::LK, t.c); t.kz = C::LK - t.kx - t.ky;
    t.lx = cart_px(C::LL, t.d); t.ly = cart_py(C::LL, t.d); t.lz = C::LL - t.lx - t.ly;
}

// per-ket-slot constants: binom(l,t) * CD^(l-t)
template <class C>
B2_HD void slot_set_cd(SlotSmem<C>& s, double CDx, double CDy, double CDz)
{
    double cd[3] = {CDx, CDy, CDz};
    for (int x = 0; x < 3; x++)
        for (int l = 0; l <= C::LL; l++) {
            // binom(l,t) CD^(l-t), zero for t>l
            double binom = 1.0;
            for (int t = 0; t <= C::LL; t++) {
                if (t > l) { s.ccd[x][l][t] = 0.0; continue; }
                double pw = 1.0;
                for (int e = 0; e < l - t; e++) pw *= cd[x];
                s.ccd[x][l][t] = binom * pw;
                binom = binom * (l - t) / (t + 1);
            }
        }
}

// Phase A: Rys roots for primitive quartet (bp, kp).  Threads g, g+G, ... < NR of the slot.
// PrimPair::cc carries sqrt(2 pi^2.5) c_i c_j K_ij / p, so the ERI prefactor is cc_b cc_k / sqrt(p+q).
template <class C>
B2_HD void phase_roots(SlotSmem<C>& s, int g, const PrimPair& bp, const PrimPair& kp, const RysTables& tb, double omega,
                       double wsign = 1.0)
{
    double p = bp.p, q = kp.p;
    double PQx = bp.Px - kp.Px, PQy = bp.Py - kp.Py, PQz = bp.Pz - kp.Pz;
    double pq = p + q;
    double rs = rsqrt(pq);
    double ipq = rs * rs;
    double rho = p * q * ipq;
    double x = rho * (PQx * PQx + PQy * PQy + PQz * PQz);
    double pref = bp.cc * kp.cc * rs * wsign;
    double theta = 1.0;
    if (omega > 0.0) {  // erf(omega r)/r: evaluate at x*theta, u*theta, w*sqrt(theta)
        theta = omega * omega / (omega * omega + rho);
        x *= theta;
        pref *= sqrt(theta);
    }
    for (int r = g; r < C::NR; r += C::G) {
        double u, w;
        rys_root(tb, C::NR, r, x, u, w);
        s.U[0][r] = u * theta;
        s.W[0][r] = w * pref;
    }
    if (g == 0) {
        double* pc = s.pc[0];
        pc[0] = p; pc[1] = q;
        pc[2] = bp.PAx; pc[3] = bp.PAy; pc[4] = bp.PAz;
        pc[5] = kp.PAx; pc[6] = kp.PAy; pc[7] = kp.PAz;
        pc[8] = PQx; pc[9] = PQy; pc[10] = PQz;
        pc[11] = ipq;
        pc[12] = 0.5 / p; pc[13] = 0.5 / q;
    }
}

// Phase A, batched path: ONE task = root r of primitive quartet b of the batch (the caller spreads the PB*NR tasks over
// the lanes of the group).  The task of root 0 also leaves the pair constants of its primitive quartet.
template <class C>
B2_HD void phase_root_one(SlotSmem<C>& s, int b, int r, const PrimPair& bp, const PrimPair& kp, const RysTables& tb, double omega,
                          double wsign)
{
    double p = bp.p, q = kp.p;
    double PQx = bp.Px - kp.Px, PQy = bp.Py - kp.Py, PQz = bp.Pz - kp.Pz;
    double pq = p + q;
    double rs = rsqrt(pq);
    double ipq = rs * rs;
    double rho = p * q * ipq;
    double x = rho * (PQx * PQx + PQy * PQy + PQz * PQz);
    double pref = bp.cc * kp.cc * rs * wsign;
    double theta = 1.0;
    if (omega > 0.0) {
        theta = omega * omega / (omega * omega + rho);
        x *= theta;
        pref *= sqrt(theta);
    }
    double u, w;
    rys_root(tb, C::NR, r, x, u, w);
    s.U[b][r] = u * theta;
    s.W[b][r] = w * pref;
    if (r == 0) {
        double* pc = s.pc[b];
        pc[0] = p; pc[1] = q;
        pc[2] = bp.PAx; pc[3] = bp.PAy; pc[4] = bp.PAz;
        pc[5] = kp.PAx; pc[6] = kp.PAy; pc[7] = kp.PAz;
        pc[8] = PQx; pc[9] = PQy; pc[10] = PQz;
        pc[11] = ipq;
        pc[12] = 0.5 / p; pc[13] = 0.5 / q;
    }
}

// Phase B: tasks (root r, direction x) = g, g+G, ... < 3*NR: vertical recurrence in registers, then the ket transfer
//   H(n; k,l) = sum_t binom(l,t) CD^(l-t) I(n, k+t)
// so that phase D only loads one contiguous row of n per direction.
template <class C>
B2_HD void vrr_one(SlotSmem<C>& s, int b, int r, int x)
{
    const double* pc = s.pc[b];
    double p = pc[0], q = pc[1];
    double ipq = pc[11];
    double hip = pc[12], hiq = pc[13];
    {
        double u = s.U[b][r];
        double b00 = 0.5 * u * ipq;
        double b10 = (1.0 - u * q * ipq) * hip;
        double b01 = (1.0 - u * p * ipq) * hiq;
        double c00 = pc[2 + x] - u * q * ipq * pc[8 + x];
        double c0p = pc[5 + x] + u * p * ipq * pc[8 + x];
        double I[C::NB1][C::NT1];
        double i0 = (x == 2) ? s.W[b][r] : 1.0;
        I[0][0] = i0;
        if (C::LB > 0) {
            I[1][0] = c00 * i0;
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
        double* H = s.H[b][x][r];
        B2_UNROLL
        for (int l = 0; l <= C::LL; l++) {
            double cf[C::LL + 1];
            B2_UNROLL
            for (int t = 0; t <= C::LL; t++) cf[t] = s.ccd[x][l][t];
            B2_UNROLL
            for (int k = 0; k <= C::LK; k++) {
                B2_UNROLL
                for (int n = 0; n <= C::LB; n++) {
                    double acc = 0.0;
                    B2_UNROLL
                    for (int t = 0; t <= l; t++) acc += cf[t] * I[n][k + t];
                    H[(l * (C::LK + 1) + k) * C::NB1P + n] = acc;
                }
            }
        }
    }
}

template <class C>
B2_HD void phase_vrr(SlotSmem<C>& s, int g)
{
    for (int task = g; task < 3 * C::NR; task += C::G) {
        int r = task / 3, x = task - 3 * r;
        vrr_one<C>(s, 0, r, x);
    }
}

// thread-local bra transfer (i -> j) for one direction from the row H(.; k,l): out[j*(LI+1)+i]
template <class C>
B2_HD void hrr_dir(const double* H, int k, int l, double AB, double* out)
{
    double T[C::NB1P];
    const double* row = H + (l * (C::LK + 1) + k) * C::NB1P;
#if defined(__CUDA_ARCH__)
    B2_UNROLL
    for (int n = 0; n < C::NB1P; n += 2) {
        double2 v2 = *reinterpret_cast<const double2*>(row + n);   // 16-byte aligned by construction
        T[n] = v2.x; T[n + 1] = v2.y;
    }
#else
    for (int n = 0; n < C::NB1; n++) T[n] = row[n];
#endif
    B2_UNROLL
    for (int i = 0; i <= C::LI; i++) out[i] = T[i];
    B2_UNROLL
    for (int j = 1; j <= C::LJ; j++) {
        B2_UNROLL
        for (int n = 0; n <= C::LB - j; n++) T[n] = T[n + 1] + AB * T[n];
        B2_UNROLL
        for (int i = 0; i <= C::LI; i++) out[j * C::NI1 + i] = T[i];
    }
}

template <class C, int P>
B2_HD void accumulate_part(double* v, const double* gx, const double* gy, const double* gz)
{
    B2_UNROLL
    for (int bb = 0; bb < C::NJP; bb++) {
        B2_UNROLL
        for (int a = 0; a < C::NI; a++) {
            constexpr int dummy = 0; (void)dummy;
            const int b = P * C::NJP + bb;
            const int ix = cart_px(C::LI, a), iy = cart_py(C::LI, a), iz = C::LI - ix - iy;
            const int jx = cart_px(C::LJ, b), jy = cart_py(C::LJ, b), jz = C::LJ - jx - jy;
            v[bb * C::NI + a] += gx[jx * C::NI1 + ix] * gy[jy * C::NI1 + iy] * gz[jz * C::NI1 + iz];
        }
    }
}

template <class C, int P>
struct PartDispatch {
    static B2_HD void run(int p, double* v, const double* gx, const double* gy, const double* gz)
    {
        if (p == P) accumulate_part<C, P>(v, gx, gy, gz);
        else PartDispatch<C, P + 1>::run(p, v, gx, gy, gz);
    }
};
template <class C>
struct PartDispatch<C, C::NP> {
    static B2_HD void run(int, double*, const double*, const double*, const double*) {}
};

// Phase D: every thread of the slot
template <class C>
B2_HD void phase_accumulate(const SlotSmem<C>& s, ThreadCtx<C>& t, double ABx, double ABy, double ABz, int b = 0)
{
    for (int r = 0; r < C::NR; r++) {
        double gx[C::NI1 * C::NJ1], gy[C::NI1 * C::NJ1], gz[C::NI1 * C::NJ1];
        hrr_dir<C>(s.H[b][0][r], t.kx, t.lx, ABx, gx);
        hrr_dir<C>(s.H[b][1][r], t.ky, t.ly, ABy, gy);
        hrr_dir<C>(s.H[b][2][r], t.kz, t.lz, ABz, gz);
        PartDispatch<C, 0>::run(t.p, t.v, gx, gy, gz);
    }
}

#ifdef __CUDA_ARCH__
#ifdef B2_EXPERIMENT_NORED
// tuning experiment only (tools/build_variant.sh nored "-DB2_EXPERIMENT_NORED"): the arithmetic stays alive, the reduction never
// executes — an upper bound on what the write-back costs.  Results are WRONG by construction.
__device__ __forceinline__ void red_add(double* addr, double val) { if (val == 1.2345678e301) atomicAdd(addr, val); }
#else
__device__ __forceinline__ void red_add(double* addr, double val) { atomicAdd(addr, val); }
#endif
#else
inline void red_add(double* addr, double val) { *addr += val; }
#endif

// Phase E: contract the register block with the density and flush.
//   Jacc[ij] += 2 f v D[kl] ; Jacc[kl] += 2 f v D[ij]            (J = Jacc + Jacc^T)
//   Kacc[ik] += f v D[jl] ; Kacc[il] += f v D[jk] ; Kacc[jk] += f v D[il] ; Kacc[jl] += f v D[ik]
//                                                                 (K = Kacc +/- Kacc^T)
// dmj/dmk: [n_dm][n][n] Cartesian; dmj symmetric; dmk symmetric or antisymmetric.
// read-only density loads: the non-coherent path is not ordered behind the reductions issued earlier, so the compiler
// may start them early
#if defined(__CUDA_ARCH__)
#define B2_LDG(p) __ldg(p)
#else
#define B2_LDG(p) (*(p))
#endif

// Every K element and J[kl] of a quartet collects sums from several of its lanes: K[i0+a, kc] from all lanes of the same c,
// J[kc, ld] from the NP parts, and so on (a (dd|dp) quartet has 648 K sums for 108 distinct K elements).  So the lanes do not
// reduce their sums into global memory one by one: each lane writes its DigestCfg::NE sums into the slot's scratch (the 2-D
// integral array H, dead once phase D is done), one row per sum and one column per lane, and then one lane per distinct
// element adds that element's contributors in lane order and issues ONE reduction.  Where H cannot hold all NE rows of the
// quartet's G lanes, the rows go through it in NRND rounds of RPR rows.  Rows of a lane (p, c, d):
//   [0, NI)              kik[a]  -> K[i0+a, kc]            contributors: the lanes of the same c
//   [NI, 2NI)            kil[a]  -> K[i0+a, ld]            the lanes of the same d
//   [2NI, 2NI+NJP)       kjk[bb] -> K[j0+p*NJP+bb, kc]     the lanes of the same p and c
//   [2NI+NJP, 2NI+2NJP)  kjl[bb] -> K[j0+p*NJP+bb, ld]     the lanes of the same p and d
//   2NI+2NJP             jkl     -> J[kc, ld]              the lanes of the same c and d
template <class C>
struct DigestCfg {
    static constexpr int NE = 2 * C::NI + 2 * C::NJP + 1;
    static constexpr int RPR = C::PB * 3 * C::NR * C::HSP / C::G;   // rows per round
    static constexpr int NRND = RPR > 0 ? (NE + RPR - 1) / RPR : 1;
    // row family f (the five lines above): its first row, and the distinct elements each of its rows feeds
    static B2_HD constexpr int row0(int f)
    {
        return f == 0 ? 0 : f == 1 ? C::NI : f == 2 ? 2 * C::NI : f == 3 ? 2 * C::NI + C::NJP : f == 4 ? 2 * C::NI + 2 * C::NJP : NE;
    }
    static B2_HD constexpr int nel(int f)
    {
        return f == 0 ? C::NK : f == 1 ? C::NL : f == 2 ? C::NP * C::NK : f == 3 ? C::NP * C::NL : C::NKL;
    }
};

// The J part of lane (p, c, d) for one density D: returns jkl = sum_ab v D[ij] (its row of the scratch) and adds the
// J[ij] of the bra block, which has one contributor per lane and element, to jacc (the stationary bra pair's registers,
// flushed once per CTA) or, without jacc, straight to J.  It runs before the rounds (phase_digest) in a phase of its own,
// so that its density loads are not scheduled next to theirs.
template <class C>
B2_HD double digest_j(const SlotSmem<C>& s, const ThreadCtx<C>& t, int i0, int j0, int n, const double* D, double* J,
                      double* jacc)
{
    const double dkl = 2.0 * s.fac * B2_LDG(&D[(size_t)(s.k0 + t.c) * n + s.l0 + t.d]);
    const int jb0 = j0 + t.p * C::NJP;
    double jkl = 0.0;
    B2_UNROLL
    for (int bb = 0; bb < C::NJP; bb++) {
        B2_UNROLL
        for (int a = 0; a < C::NI; a++) {
            const double val = t.v[bb * C::NI + a];
            const size_t ij = (size_t)(i0 + a) * n + (jb0 + bb);
            jkl += val * B2_LDG(&D[ij]);
            if (jacc) jacc[bb * C::NI + a] += val * dkl;
            else red_add(&J[ij], val * dkl);
        }
    }
    return jkl;
}

// Lane (p, c, d)'s sums of rows [r0, r0 + RPR), written to the slot's scratch: row r at H + (r - r0) * G + g.  The K sums
// are computed in the round that stores them, so the register block is the only state a lane carries from round to round.
// Dk: this density (null: no K of it, those rows are zero); jkl: the J row (digest_j, zero without J).
template <class C>
B2_HD void phase_digest(SlotSmem<C>& s, const ThreadCtx<C>& t, int r0, int i0, int j0, int n, const double* Dk, double jkl)
{
    using DG = DigestCfg<C>;
    static_assert(DG::RPR >= 1, "the 2-D integral array of a slot must hold one row of the quartet's lanes");
    const int r1 = r0 + DG::RPR;
    const int kc = s.k0 + t.c, ld = s.l0 + t.d;
    const int jb0 = j0 + t.p * C::NJP;
    double* X = &s.H[0][0][0][0] + t.g;
    if (!Dk) {
        B2_UNROLL
        for (int r = 0; r < DG::NE; r++)
            if (r >= r0 && r < r1) X[(r - r0) * C::G] = r == DG::NE - 1 ? jkl : 0.0;
        return;
    }
    // the density columns the rows of this round read: D[jb, ld] (kik), D[jb, kc] (kil), D[i0+a, ld] (kjk), D[i0+a, kc] (kjl)
    const auto in_round = [&](int f_) { return DG::row0(f_) < r1 && DG::row0(f_ + 1) > r0; };
    double djl[C::NJP], djk[C::NJP], dil[C::NI], dik[C::NI];
    B2_UNROLL
    for (int bb = 0; bb < C::NJP; bb++) {
        if (in_round(0)) djl[bb] = B2_LDG(&Dk[(size_t)(jb0 + bb) * n + ld]);
        if (in_round(1)) djk[bb] = B2_LDG(&Dk[(size_t)(jb0 + bb) * n + kc]);
    }
    B2_UNROLL
    for (int a = 0; a < C::NI; a++) {
        if (in_round(2)) dil[a] = B2_LDG(&Dk[(size_t)(i0 + a) * n + ld]);
        if (in_round(3)) dik[a] = B2_LDG(&Dk[(size_t)(i0 + a) * n + kc]);
    }
    B2_UNROLL
    for (int r = 0; r < DG::NE; r++) {
        if (r < r0 || r >= r1) continue;
        double sum = 0.0;
        if (r < 2 * C::NI) {                      // kik[a] = sum_b v D[jb, ld],  kil[a] = sum_b v D[jb, kc]
            const int a = r < C::NI ? r : r - C::NI;
            B2_UNROLL
            for (int bb = 0; bb < C::NJP; bb++) sum += t.v[bb * C::NI + a] * (r < C::NI ? djl[bb] : djk[bb]);
        } else if (r < 2 * C::NI + 2 * C::NJP) {  // kjk[b] = sum_a v D[i0+a, ld],  kjl[b] = sum_a v D[i0+a, kc]
            const int bb = r < 2 * C::NI + C::NJP ? r - 2 * C::NI : r - 2 * C::NI - C::NJP;
            B2_UNROLL
            for (int a = 0; a < C::NI; a++) sum += t.v[bb * C::NI + a] * (r < 2 * C::NI + C::NJP ? dil[a] : dik[a]);
        } else {
            sum = jkl;
        }
        X[(r - r0) * C::G] = sum;
    }
}

// the distinct elements fed by rows [r0, r0 + RPR), tasks g, g + G, ... of the quartet: each sums its contributors in lane
// order and issues one reduction.  J / K: the outputs of this density (null: not computed).
template <class C>
B2_HD void digest_flush(const SlotSmem<C>& s, int g, int r0, int i0, int j0, int n, double* J, double* K)
{
    using DG = DigestCfg<C>;
    const int r1 = r0 + DG::RPR < DG::NE ? r0 + DG::RPR : DG::NE;
    const double* X = &s.H[0][0][0][0];
    const double f = s.fac;
    const int k0 = s.k0, l0 = s.l0;
    B2_UNROLL
    for (int fam = 0; fam < 5; fam++) {
        const int lo = DG::row0(fam) > r0 ? DG::row0(fam) : r0;
        const int hi = DG::row0(fam + 1) < r1 ? DG::row0(fam + 1) : r1;
        if (hi <= lo || (fam < 4 ? K : J) == nullptr) continue;
        const int nel = DG::nel(fam);
        for (int task = g; task < (hi - lo) * nel; task += C::G) {
            const int row = lo + task / nel, el = task - (task / nel) * nel;
            const double* x = X + (row - r0) * C::G;
            double sum = 0.0;
            if (fam == 0) {          // K[i0+a, kc], c = el: lanes p*NKL + d*NK + c
                B2_UNROLL
                for (int p = 0; p < C::NP; p++) {
                    B2_UNROLL
                    for (int d = 0; d < C::NL; d++) sum += x[p * C::NKL + d * C::NK + el];
                }
                red_add(&K[(size_t)(i0 + row) * n + k0 + el], f * sum);
            } else if (fam == 1) {   // K[i0+a, ld], d = el
                B2_UNROLL
                for (int p = 0; p < C::NP; p++) {
                    B2_UNROLL
                    for (int c = 0; c < C::NK; c++) sum += x[p * C::NKL + el * C::NK + c];
                }
                red_add(&K[(size_t)(i0 + row - C::NI) * n + l0 + el], f * sum);
            } else if (fam == 2) {   // K[j0+p*NJP+bb, kc], el = p*NK + c
                const int p = el / C::NK, c = el - p * C::NK;
                B2_UNROLL
                for (int d = 0; d < C::NL; d++) sum += x[p * C::NKL + d * C::NK + c];
                red_add(&K[(size_t)(j0 + p * C::NJP + row - 2 * C::NI) * n + k0 + c], f * sum);
            } else if (fam == 3) {   // K[j0+p*NJP+bb, ld], el = p*NL + d
                const int p = el / C::NL, d = el - p * C::NL;
                B2_UNROLL
                for (int c = 0; c < C::NK; c++) sum += x[p * C::NKL + d * C::NK + c];
                red_add(&K[(size_t)(j0 + p * C::NJP + row - 2 * C::NI - C::NJP) * n + l0 + d], f * sum);
            } else {                 // J[kc, ld], el = d*NK + c
                B2_UNROLL
                for (int p = 0; p < C::NP; p++) sum += x[p * C::NKL + el];
                red_add(&J[(size_t)(k0 + el % C::NK) * n + l0 + el / C::NK], 2.0 * f * sum);
            }
        }
    }
}

// Phase E without the scratch: every lane reduces its own sums straight into J and K (the classes of
// class_reduces_per_lane).
template <class C>
B2_HD void phase_digest_lane(const SlotSmem<C>& s, const ThreadCtx<C>& t, int i0, int j0, int n, int n_dm,
                        const double* dmj, const double* dmk, double* vj, double* vk, double* jacc)
{
    const double f = s.fac;
    const int kc = s.k0 + t.c, ld = s.l0 + t.d;
    const int b0 = t.p * C::NJP;
    const size_t n2 = (size_t)n * n;
    for (int idm = 0; idm < n_dm; idm++) {
        if (vj) {
            const double* D = dmj + idm * n2;
            double* J = vj + idm * n2;
            double dkl = 2.0 * f * B2_LDG(&D[(size_t)kc * n + ld]);
            double jkl = 0.0;
            B2_UNROLL
            for (int bb = 0; bb < C::NJP; bb++) {
                B2_UNROLL
                for (int a = 0; a < C::NI; a++) {
                    double val = t.v[bb * C::NI + a];
                    size_t ij = (size_t)(i0 + a) * n + (j0 + b0 + bb);
                    jkl += val * B2_LDG(&D[ij]);
                    if (jacc) jacc[bb * C::NI + a] += val * dkl;  // stationary bra pair: flushed once per CTA
                    else red_add(&J[ij], val * dkl);
                }
            }
            red_add(&J[(size_t)kc * n + ld], 2.0 * f * jkl);
        }
        if (vk) {
            const double* D = dmk + idm * n2;
            double* K = vk + idm * n2;
            double kjk[C::NJP], kjl[C::NJP];
            double kik[C::NI], kil[C::NI];
            double dik[C::NI], dil[C::NI];
            B2_UNROLL
            for (int a = 0; a < C::NI; a++) {
                kik[a] = 0.0; kil[a] = 0.0;
                dik[a] = B2_LDG(&D[(size_t)(i0 + a) * n + kc]);
                dil[a] = B2_LDG(&D[(size_t)(i0 + a) * n + ld]);
            }
            B2_UNROLL
            for (int bb = 0; bb < C::NJP; bb++) {
                int jb = j0 + b0 + bb;
                double djl = B2_LDG(&D[(size_t)jb * n + ld]), djk = B2_LDG(&D[(size_t)jb * n + kc]);
                double sjk = 0.0, sjl = 0.0;
                B2_UNROLL
                for (int a = 0; a < C::NI; a++) {
                    double val = t.v[bb * C::NI + a];
                    kik[a] += val * djl;
                    kil[a] += val * djk;
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
            for (int bb = 0; bb < C::NJP; bb++) {
                int jb = j0 + b0 + bb;
                red_add(&K[(size_t)jb * n + kc], f * kjk[bb]);
                red_add(&K[(size_t)jb * n + ld], f * kjl[bb]);
            }
        }
    }
}

// Screening decision of CVHFnrs8_prescreen (pyscf/lib/vhf/optimizer.c:90-117) on device shells.
B2_HD bool keep_quartet(double qij, double qkl, int ish, int jsh, int ksh, int lsh, const double* dmc, int nsh,
                        double tol, bool do_j, bool do_k)
{
    double qq = qij * qkl;
    if (!(qq > tol)) return false;
    double dmin = tol / qq;
    bool keep = false;
    if (do_j) keep = (4.0 * dmc[ish * nsh + jsh] > dmin) || (4.0 * dmc[ksh * nsh + lsh] > dmin);
    if (do_k && !keep)
        keep = (dmc[jsh * nsh + ksh] > dmin) || (dmc[jsh * nsh + lsh] > dmin) || (dmc[ish * nsh + ksh] > dmin) ||
               (dmc[ish * nsh + lsh] > dmin);
    return keep;
}

// ---------------------------------------------------------------------------------------------
// Generic (run-time angular momentum) diagonal integrals for the Schwarz bounds:
//   q = sqrt(max_ab |(ab|ab)|)   <- CVHFnr_int2e_q_cond, pyscf/lib/vhf/optimizer.c:408-454
B2_HD double schwarz_pair(int la, int lb, const ShellPair& sp, const PrimPair* prims, const RysTables& tb, double omega)
{
    const int L = la + lb;          // per side
    const int nr = L + 1;           // (2L)/2 + 1
    const int na = ncart(la), nb = ncart(lb);
    double acc[ncart(LMAX) * ncart(LMAX)];
    for (int e = 0; e < na * nb; e++) acc[e] = 0.0;
    double AB[3] = {sp.ABx, sp.ABy, sp.ABz};
    for (int ip = 0; ip < sp.nprim; ip++)
        for (int kp = 0; kp < sp.nprim; kp++) {
            const PrimPair& bp = prims[sp.prim_off + ip];
            const PrimPair& kq = prims[sp.prim_off + kp];
            double p = bp.p, q = kq.p, pq = p + q, ipq = 1.0 / pq;
            double PQ[3] = {bp.Px - kq.Px, bp.Py - kq.Py, bp.Pz - kq.Pz};
            double PA[3] = {bp.PAx, bp.PAy, bp.PAz}, QC[3] = {kq.PAx, kq.PAy, kq.PAz};
            double rho = p * q * ipq;
            double x = rho * (PQ[0] * PQ[0] + PQ[1] * PQ[1] + PQ[2] * PQ[2]);
            double pref = bp.cc * kq.cc / sqrt(pq);
            // omega < 0: erfc(|omega| r)/r = 1/r - erf(|omega| r)/r, i.e. a second root set with negated weights
            const double x0 = x, pref0 = pref;
            for (int r2 = 0; r2 < (omega < 0.0 ? 2 * nr : nr); r2++) {
                const int r = r2 % nr;
                double theta = 1.0;
                x = x0; pref = pref0;
                const double om = (omega < 0.0) ? (r2 >= nr ? -omega : 0.0) : omega;
                if (om > 0.0) { theta = om * om / (om * om + rho); x *= theta; pref *= sqrt(theta); }
                if (r2 >= nr) pref = -pref;
                double u, w;
                rys_root(tb, nr, r, x, u, w);
                u *= theta; w *= pref;
                double I[3][2 * LMAX + 1][2 * LMAX + 1];
                double b00 = 0.5 * u * ipq, b10 = (1.0 - u * q * ipq) * 0.5 / p, b01 = (1.0 - u * p * ipq) * 0.5 / q;
                for (int d = 0; d < 3; d++) {
                    double c00 = PA[d] - u * q * ipq * PQ[d], c0p = QC[d] + u * p * ipq * PQ[d];
                    I[d][0][0] = (d == 2) ? w : 1.0;
                    if (L > 0) I[d][1][0] = c00 * I[d][0][0];
                    for (int n = 1; n < L; n++) I[d][n + 1][0] = c00 * I[d][n][0] + n * b10 * I[d][n - 1][0];
                    for (int m = 0; m < L; m++)
                        for (int n = 0; n <= L; n++) {
                            double val = c0p * I[d][n][m];
                            if (m > 0) val += m * b01 * I[d][n][m - 1];
                            if (n > 0) val += n * b00 * I[d][n - 1][m];
                            I[d][n][m + 1] = val;
                        }
                }
                for (int b = 0; b < nb; b++)
                    for (int a = 0; a < na; a++) {
                        int ia[3] = {cart_px(la, a), cart_py(la, a), 0};
                        ia[2] = la - ia[0] - ia[1];
                        int jb[3] = {cart_px(lb, b), cart_py(lb, b), 0};
                        jb[2] = lb - jb[0] - jb[1];
                        double prod = 1.0;
                        for (int d = 0; d < 3; d++) {
                            // G(i,j,i,j) = sum_s sum_t C(j,s)C(j,t) AB^(2j-s-t) I[i+s][i+t]
                            double gsum = 0.0;
                            double bs = 1.0;
                            for (int s_ = 0; s_ <= jb[d]; s_++) {
                                double ps = 1.0;
                                for (int e = 0; e < jb[d] - s_; e++) ps *= AB[d];
                                double bt = 1.0;
                                for (int t_ = 0; t_ <= jb[d]; t_++) {
                                    double pt = 1.0;
                                    for (int e = 0; e < jb[d] - t_; e++) pt *= AB[d];
                                    gsum += bs * ps * bt * pt * I[d][ia[d] + s_][ia[d] + t_];
                                    bt = bt * (jb[d] - t_) / (t_ + 1);
                                }
                                bs = bs * (jb[d] - s_) / (s_ + 1);
                            }
                            prod *= gsum;
                        }
                        acc[b * na + a] += prod;
                    }
            }
        }
    double m = 0.0;
    for (int e = 0; e < na * nb; e++) m = fmax(m, fabs(acc[e]));
    return sqrt(m);
}

// The same bound in the REFERENCE's normalisation: q = sqrt(max_{A,B} |(AB|AB)|) over the real-spherical functions A of shell a
// and B of shell b, exactly what CVHFnr_int2e_q_cond (pyscf/lib/vhf/optimizer.c:408-454) takes from int2e_sph.  The Cartesian
// block M[ab][a'b'] = (ab|a'b') is accumulated over primitives and roots, then every spherical pair is u^T M u with
// u = T_a[A,:] (x) T_b[B,:] (T = the cart->sph matrices the density / J,K transforms use).  Setup only: one thread per shell pair,
// M in thread-local memory (100 x 100 doubles for an (ff| pair).
B2_HD double schwarz_pair_sph(int la, int lb, const ShellPair& sp, const PrimPair* prims, const RysTables& tb, double omega,
                              const double* Ta, const double* Tb, double* M, int nfa, int nfb)   // nfa, nfb: rows of Ta, Tb
{
    const int L = la + lb, nr = L + 1;
    const int na = ncart(la), nb = ncart(lb), ne = na * nb;
    for (int e = 0; e < ne * ne; e++) M[e] = 0.0;
    const double AB[3] = {sp.ABx, sp.ABy, sp.ABz};
    for (int ip = 0; ip < sp.nprim; ip++)
        for (int kp = 0; kp < sp.nprim; kp++) {
            const PrimPair& bp = prims[sp.prim_off + ip];
            const PrimPair& kq = prims[sp.prim_off + kp];
            double p = bp.p, q = kq.p, pq = p + q, ipq = 1.0 / pq;
            double PQ[3] = {bp.Px - kq.Px, bp.Py - kq.Py, bp.Pz - kq.Pz};
            double PA[3] = {bp.PAx, bp.PAy, bp.PAz}, QC[3] = {kq.PAx, kq.PAy, kq.PAz};
            double rho = p * q * ipq;
            const double x0 = rho * (PQ[0] * PQ[0] + PQ[1] * PQ[1] + PQ[2] * PQ[2]), pref0 = bp.cc * kq.cc / sqrt(pq);
            for (int r2 = 0; r2 < (omega < 0.0 ? 2 * nr : nr); r2++) {
                const int r = r2 % nr;
                double theta = 1.0, x = x0, pref = pref0;
                const double om = (omega < 0.0) ? (r2 >= nr ? -omega : 0.0) : omega;
                if (om > 0.0) { theta = om * om / (om * om + rho); x *= theta; pref *= sqrt(theta); }
                if (r2 >= nr) pref = -pref;
                double u, w;
                rys_root(tb, nr, r, x, u, w);
                u *= theta; w *= pref;
                double I[3][2 * LMAX + 1][2 * LMAX + 1];
                double b00 = 0.5 * u * ipq, b10 = (1.0 - u * q * ipq) * 0.5 / p, b01 = (1.0 - u * p * ipq) * 0.5 / q;
                // G[d][(i*(lb+1)+j)*nij + (i'*(lb+1)+j')] = 2-D integral of direction d with bra powers (i,j), ket powers (i',j')
                double G[3][16 * 16];
                const int nij = (la + 1) * (lb + 1);
                for (int d = 0; d < 3; d++) {
                    double c00 = PA[d] - u * q * ipq * PQ[d], c0p = QC[d] + u * p * ipq * PQ[d];
                    I[d][0][0] = (d == 2) ? w : 1.0;
                    if (L > 0) I[d][1][0] = c00 * I[d][0][0];
                    for (int n = 1; n < L; n++) I[d][n + 1][0] = c00 * I[d][n][0] + n * b10 * I[d][n - 1][0];
                    for (int m = 0; m < L; m++)
                        for (int n = 0; n <= L; n++) {
                            double val = c0p * I[d][n][m];
                            if (m > 0) val += m * b01 * I[d][n][m - 1];
                            if (n > 0) val += n * b00 * I[d][n - 1][m];
                            I[d][n][m + 1] = val;
                        }
                    for (int i = 0; i <= la; i++)
                        for (int j = 0; j <= lb; j++)
                            for (int i2 = 0; i2 <= la; i2++)
                                for (int j2 = 0; j2 <= lb; j2++) {
                                    double gsum = 0.0, bs = 1.0;
                                    for (int s_ = 0; s_ <= j; s_++) {
                                        double ps = 1.0;
                                        for (int e = 0; e < j - s_; e++) ps *= AB[d];
                                        double bt = 1.0;
                                        for (int t_ = 0; t_ <= j2; t_++) {
                                            double pt = 1.0;
                                            for (int e = 0; e < j2 - t_; e++) pt *= AB[d];
                                            gsum += bs * ps * bt * pt * I[d][i + s_][i2 + t_];
                                            bt = bt * (j2 - t_) / (t_ + 1);
                                        }
                                        bs = bs * (j - s_) / (s_ + 1);
                                    }
                                    G[d][(i * (lb + 1) + j) * nij + i2 * (lb + 1) + j2] = gsum;
                                }
                }
                for (int b = 0; b < nb; b++)
                    for (int a = 0; a < na; a++) {
                        const int ax = cart_px(la, a), ay = cart_py(la, a), az = la - ax - ay;
                        const int bx = cart_px(lb, b), by = cart_py(lb, b), bz = lb - bx - by;
                        const int rx = (ax * (lb + 1) + bx) * nij, ry = (ay * (lb + 1) + by) * nij, rz = (az * (lb + 1) + bz) * nij;
                        double* Mrow = M + (size_t)(b * na + a) * ne;
                        for (int b2 = 0; b2 < nb; b2++)
                            for (int a2 = 0; a2 < na; a2++) {
                                const int cx = cart_px(la, a2), cy = cart_py(la, a2), cz = la - cx - cy;
                                const int dx = cart_px(lb, b2), dy = cart_py(lb, b2), dz = lb - dx - dy;
                                Mrow[b2 * na + a2] += G[0][rx + cx * (lb + 1) + dx] * G[1][ry + cy * (lb + 1) + dy] * G[2][rz + cz * (lb + 1) + dz];
                            }
                    }
            }
        }
    double best = 0.0;
    for (int A = 0; A < nfa; A++)
        for (int B = 0; B < nfb; B++) {
            double val = 0.0;
            for (int b = 0; b < nb; b++)
                for (int a = 0; a < na; a++) {
                    const double ue = Ta[A * na + a] * Tb[B * nb + b];
                    if (ue == 0.0) continue;
                    const double* Mrow = M + (size_t)(b * na + a) * ne;
                    double acc = 0.0;
                    for (int b2 = 0; b2 < nb; b2++)
                        for (int a2 = 0; a2 < na; a2++) acc += Mrow[b2 * na + a2] * Ta[A * na + a2] * Tb[B * nb + b2];
                    val += ue * acc;
                }
            best = fmax(best, fabs(val));
        }
    return sqrt(best);
}

}  // namespace b200jk
