// host_common.hpp — backend layer (CUDA runtime or CPU emulation), handle definition and small host helpers
// shared by b200jk.cu (4-center path) and df.cu (density-fitting path).
#pragma once
#include "../../include/b200jk.h"

#include <algorithm>
#include <chrono>
#include <cmath>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <stdexcept>
#include <string>
#include <vector>

#include "jk_block.cuh"

using namespace b200jk;

extern "C" const unsigned char b200jk_rys_blob[];
extern "C" const unsigned int b200jk_rys_blob_size;

// ------------------------------------------------------------------------------------------------
// backend: CUDA runtime or CPU emulation
#ifndef B200JK_EMULATE
#include <cuda_runtime.h>
#define CK(call)                                                                                       \
    do {                                                                                               \
        cudaError_t e_ = (call);                                                                       \
        if (e_ != cudaSuccess) {                                                                       \
            char buf_[512];                                                                            \
            snprintf(buf_, sizeof buf_, "%s failed: %s (%s:%d)", #call, cudaGetErrorString(e_), __FILE__, __LINE__); \
            throw std::runtime_error(buf_);                                                            \
        }                                                                                              \
    } while (0)
static void* dev_alloc(size_t n) { void* p = nullptr; CK(cudaMalloc(&p, n ? n : 8)); return p; }
static void dev_free(void* p) { if (p) cudaFree(p); }
static void h2d(void* d, const void* h, size_t n, cudaStream_t s = 0) { CK(cudaMemcpyAsync(d, h, n, cudaMemcpyHostToDevice, s)); }
static void d2h(void* h, const void* d, size_t n, cudaStream_t s = 0) { CK(cudaMemcpyAsync(h, d, n, cudaMemcpyDeviceToHost, s)); }
static void dev_zero(void* d, size_t n, cudaStream_t s = 0) { CK(cudaMemsetAsync(d, 0, n, s)); }
static void dev_sync() { CK(cudaDeviceSynchronize()); }
template <class F>
__global__ void generic_kernel(long n, F f)
{
    long i = blockIdx.x * (long)blockDim.x + threadIdx.x;
    if (i < n) f(i);
}
template <class F>
static void launch_1d(long n, const F& f, cudaStream_t s = 0)
{
    if (n <= 0) return;
    generic_kernel<F><<<(unsigned)((n + 127) / 128), 128, 0, s>>>(n, f);
    CK(cudaGetLastError());
}
typedef cudaStream_t stream_t;
#else
#include <stdexcept>
static void* dev_alloc(size_t n) { return calloc(1, n ? n : 8); }
static void dev_free(void* p) { free(p); }
typedef int stream_t;
static void h2d(void* d, const void* h, size_t n, stream_t = 0) { memcpy(d, h, n); }
static void d2h(void* h, const void* d, size_t n, stream_t = 0) { memcpy(h, d, n); }
static void dev_zero(void* d, size_t n, stream_t = 0) { memset(d, 0, n); }
static void dev_sync() {}
template <class F>
static void launch_1d(long n, const F& f, stream_t = 0)
{
    for (long i = 0; i < n; i++) f(i);
}
#endif
#include <stdexcept>

// ------------------------------------------------------------------------------------------------
namespace b2host {

constexpr int ATM_SLOTS = 6, BAS_SLOTS = 8, ATOM_OF = 0, ANG_OF = 1, NPRIM_OF = 2, NCTR_OF = 3, PTR_EXP = 5, PTR_COEFF = 6,
              PTR_COORD = 1;
constexpr int LAO_MAX = 3;                                 // orbital shells up to f on the 4-center path
constexpr int NPC = (LAO_MAX + 1) * (LAO_MAX + 2) / 2;     // pair classes
constexpr double PRIM_CUT = 1e-18;                         // drop primitive pairs with |cc| below this

struct DevShell {
    int l, nprim, ref_shell, sph_off, cart_off;
    double r[3];
    std::vector<double> e, c;
};

struct PairClass {
    int la = 0, lb = 0;
    std::vector<ShellPair> all;      // every pair, unsorted, q not set
    std::vector<ShellPair> kept;     // screened, deeply contracted pairs split into sub-pairs, sorted (block kernels)
    ShellPair* d_all = nullptr;
    ShellPair* d_kept = nullptr;
};

inline double binom(int n, int k)
{
    if (k < 0 || k > n) return 0.0;
    double r = 1.0;
    for (int i = 1; i <= k; i++) r = r * (n - k + i) / i;
    return r;
}
inline double fact(int n) { double r = 1; for (int i = 2; i <= n; i++) r *= i; return r; }
inline int cart_index(int l, int lx, int ly)
{
    int idx = 0;
    for (int x = l; x > lx; x--) idx += l - x + 1;
    return idx + (l - lx - ly);
}
// Real solid harmonics (orthonormal on the sphere) in terms of Cartesian monomials, libcint order
// (p: x,y,z ; l>=2: m=-l..l).  Helgaker, Jorgensen, Olsen, "Molecular Electronic-Structure Theory", eq. 6.4.47.
// Cartesian AOs (mol.cart = True): libcint's Cartesian functions are the bare monomials times the radial part, with the
// s and p angular factors it also puts into the spherical functions (pyscf/gto/mole.py:159-181): T = fac(l) * identity
inline std::vector<double> make_c2c(int l)
{
    int nc = ncart(l);
    std::vector<double> T((size_t)nc * nc, 0.0);
    const double f = l == 0 ? 0.282094791773878143 : (l == 1 ? 0.488602511902919921 : 1.0);
    for (int i = 0; i < nc; i++) T[(size_t)i * nc + i] = f;
    return T;
}
inline std::vector<double> make_c2s(int l)
{
    int nc = ncart(l), ns = 2 * l + 1;
    std::vector<double> T((size_t)ns * nc, 0.0);
    if (l == 0) { T[0] = 0.282094791773878143; return T; }
    if (l == 1) { for (int i = 0; i < 3; i++) T[i * 3 + i] = 0.488602511902919921; return T; }
    double ang = std::sqrt((2 * l + 1) / (4.0 * M_PI));
    for (int m = -l; m <= l; m++) {
        int am = std::abs(m);
        double N = 1.0 / (std::pow(2.0, am) * fact(l)) * std::sqrt(2.0 * fact(l + am) * fact(l - am) / (m == 0 ? 2.0 : 1.0));
        int two_vm = (m < 0) ? 1 : 0;
        for (int t = 0; t <= (l - am) / 2; t++)
            for (int u = 0; u <= t; u++) {
                int vmax2 = 2 * (int)std::floor(am / 2.0 - two_vm / 2.0) + two_vm;
                for (int two_v = two_vm; two_v <= vmax2; two_v += 2) {
                    int sp = t + (two_v - two_vm) / 2;
                    double Cf = ((sp & 1) ? -1.0 : 1.0) * std::pow(0.25, t) * binom(l, t) * binom(l - t, am + t) *
                                binom(t, u) * binom(am, two_v);
                    int lx = 2 * t + am - 2 * u - two_v, ly = 2 * u + two_v, lz = l - 2 * t - am;
                    if (lx < 0 || ly < 0 || lz < 0) continue;
                    T[(size_t)(m + l) * nc + cart_index(l, lx, ly)] += ang * N * Cf;
                }
            }
    }
    return T;
}

}  // namespace b2host
using namespace b2host;

struct DFState;

struct b200jk_handle_s {
    int device = 0;
    std::string err;
    std::vector<DevShell> sh;
    int nsh = 0, ncart = 0, nsph = 0, nbas_ref = 0;
    int cart = 0;        // 1: Cartesian AOs (mol.cart = True): "spherical" index space = the ncart(l) libcint Cartesian functions of each shell
    std::vector<PrimPair> prims;
    PrimPair* d_prims = nullptr;
    PairClass pc[NPC];
    double* d_rys = nullptr;
    RysTables tb{nullptr, nullptr};
    // AO transform tables
    int *d_cart_sh = nullptr, *d_cart_comp = nullptr, *d_sph_sh = nullptr, *d_sph_m = nullptr;
    int *d_sh_l = nullptr, *d_sh_cart = nullptr, *d_sh_sph = nullptr;
    double* d_c2s = nullptr;
    int c2s_off[LMAX + 2] = {0};
    int* d_c2s_off = nullptr;
    std::vector<int> ref_shell_of;  // device shell -> reference shell
    double tol = 1e-13, omega = 0.0;
    bool screened = false;
    // workspaces
    size_t ws_ndm = 0;
    double *d_dm_sph = nullptr, *d_out_sph = nullptr, *d_dmj = nullptr, *d_dmk = nullptr, *d_vj = nullptr, *d_vk = nullptr,
           *d_dmc = nullptr;
    unsigned long long* d_counters = nullptr;
    b200jk_stats stats{};
#ifndef B200JK_EMULATE
    cudaStream_t stream = nullptr;
    cudaStream_t own_stream = nullptr;
    cudaEvent_t ev0 = nullptr, ev1 = nullptr;
    std::vector<cudaEvent_t> cls_ev;
    std::vector<cudaStream_t> side;      // class kernels are spread over side streams (small classes overlap)
    std::vector<cudaEvent_t> side_ev;
    cudaEvent_t ev_in = nullptr;
#endif
    int profile = 0;
    int shard_rank = 0, shard_world = 1;   // multi-GPU work partition (b200jk_set_shard)
    DFState* df = nullptr;          // density-fitting state (df.cu)
    void (*df_free)(DFState*) = nullptr;
    int df_dev_rows = -1;           // b200jk_df_set_device_rows: cap on the tensor rows kept in HBM (-1: automatic)
    double class_ms[NPC * NPC] = {0};
    double class_cost[NPC * NPC] = {0};   // measured class times handed in by the caller (b200jk_set_class_costs); 0 = use the model
    bool have_costs = false;
    // in-core path (mf._eri): the stored two-electron integrals, 8-fold / 4-fold packed or full (b200jk_incore_set_eri)
    double* d_eri = nullptr; long neri = 0; int eri_sym = 0;
};


namespace b2host {

// ------------------------------------------------------------------------------------------------
// small kernels (functors so that the same code runs under emulation)
struct SchwarzFn {
    ShellPair* pairs; const PrimPair* prims; RysTables tb; double omega; int la, lb;
    B2_HD void operator()(long i) const { pairs[i].q = schwarz_pair(la, lb, pairs[i], prims, tb, omega); }
};
// the reference's Schwarz bound (normalised real-spherical functions); scratch: (ncart(la) ncart(lb))^2 doubles per pair
struct SchwarzSphFn {
    ShellPair* pairs; const PrimPair* prims; RysTables tb; double omega; int la, lb; const double *Ta, *Tb; double* scratch; int nfa, nfb;
    B2_HD void operator()(long i) const
    {
        const long ne = (long)((la + 1) * (la + 2) / 2) * ((lb + 1) * (lb + 2) / 2);
        pairs[i].q = schwarz_pair_sph(la, lb, pairs[i], prims, tb, omega, Ta, Tb, scratch + i * ne * ne, nfa, nfb);
    }
};

// D_cart[s][mu][nu] = sum_{m,m'} T[m,mu] Dsym[m,m'] T[m',nu]; mode 0: (D+D^T)/2, 1: (D-D^T)/2, 2: D as is
struct Sph2CartFn {
    const double* dsph; double* dcart; int nsph, ncart, mode;
    const int *cart_sh, *cart_comp, *sh_l, *sh_sph, *c2s_off; const double* c2s; int cart = 0;
    B2_HD void operator()(long idx) const
    {
        long n2 = (long)ncart * ncart;
        int s = (int)(idx / n2);
        long rem = idx - s * n2;
        int mu = (int)(rem / ncart), nu = (int)(rem - (long)mu * ncart);
        int sa = cart_sh[mu], sb = cart_sh[nu];
        int la = sh_l[sa], lb = sh_l[sb];
        int nca = ncart_rt(la), ncb = ncart_rt(lb);
        const double* Ta = c2s + c2s_off[la] + cart_comp[mu];
        const double* Tb = c2s + c2s_off[lb] + cart_comp[nu];
        const double* D = dsph + (size_t)s * nsph * nsph;
        int oa = sh_sph[sa], ob = sh_sph[sb];
        double acc = 0.0;
        const int nfa = cart ? nca : 2 * la + 1, nfb = cart ? ncb : 2 * lb + 1;   // functions per shell in the caller's AO basis
        for (int m = 0; m < nfa; m++) {
            double ta = Ta[m * nca];
            if (ta == 0.0) continue;
            for (int mp = 0; mp < nfb; mp++) {
                double tb_ = Tb[mp * ncb];
                if (tb_ == 0.0) continue;
                double d1 = D[(size_t)(oa + m) * nsph + ob + mp], d2 = D[(size_t)(ob + mp) * nsph + oa + m];
                double d = (mode == 0) ? 0.5 * (d1 + d2) : (mode == 1 ? 0.5 * (d1 - d2) : d1);
                acc += ta * tb_ * d;
            }
        }
        dcart[idx] = acc;
    }
    static B2_HD int ncart_rt(int l) { return (l + 1) * (l + 2) / 2; }
};

// out_sph[s][m][m'] (+)= sum T[m,mu] (X[mu,nu] + sign*X[nu,mu]) T[m',nu]
struct Cart2SphFn {
    const double* xcart; double* osph; int nsph, ncart; double sign; int accumulate;
    const int *sph_sh, *sph_m, *sh_l, *sh_cart, *c2s_off; const double* c2s;
    B2_HD void operator()(long idx) const
    {
        long n2 = (long)nsph * nsph;
        int s = (int)(idx / n2);
        long rem = idx - s * n2;
        int a = (int)(rem / nsph), b = (int)(rem - (long)a * nsph);
        int sa = sph_sh[a], sb = sph_sh[b];
        int la = sh_l[sa], lb = sh_l[sb];
        int nca = (la + 1) * (la + 2) / 2, ncb = (lb + 1) * (lb + 2) / 2;
        const double* Ta = c2s + c2s_off[la] + sph_m[a] * nca;
        const double* Tb = c2s + c2s_off[lb] + sph_m[b] * ncb;
        const double* X = xcart + (size_t)s * ncart * ncart;
        int oa = sh_cart[sa], ob = sh_cart[sb];
        double acc = 0.0;
        for (int c = 0; c < nca; c++) {
            double ta = Ta[c];
            if (ta == 0.0) continue;
            for (int d = 0; d < ncb; d++) {
                double tb_ = Tb[d];
                if (tb_ == 0.0) continue;
                acc += ta * tb_ * (X[(size_t)(oa + c) * ncart + ob + d] + sign * X[(size_t)(ob + d) * ncart + oa + c]);
            }
        }
        if (accumulate) osph[idx] += acc; else osph[idx] = acc;
    }
};

// dm_cond as the reference defines it (CVHFnr_dm_cond, pyscf/lib/vhf/optimizer.c:494-518): (|D_mn| + |D_nm|)/2 maximised over the
// SPHERICAL block of the two (device) shells and over all density matrices — the scale the spherical Schwarz bounds live on
struct DmCondSphFn {
    const double* dsph; int nd; double* dmc; int nsh, nsph; const int *sh_l, *sh_sph; int cart = 0;
    B2_HD void operator()(long idx) const
    {
        int i = (int)(idx / nsh), j = (int)(idx - (long)i * nsh);
        int ni = cart ? (sh_l[i] + 1) * (sh_l[i] + 2) / 2 : 2 * sh_l[i] + 1, nj = cart ? (sh_l[j] + 1) * (sh_l[j] + 2) / 2 : 2 * sh_l[j] + 1;
        double m = 0.0;
        for (int s = 0; s < nd; s++) {
            const double* D = dsph + (size_t)s * nsph * nsph;
            for (int a = 0; a < ni; a++)
                for (int b = 0; b < nj; b++) {
                    double v = 0.5 * (fabs(D[(size_t)(sh_sph[i] + a) * nsph + sh_sph[j] + b]) + fabs(D[(size_t)(sh_sph[j] + b) * nsph + sh_sph[i] + a]));
                    m = v > m ? v : m;
                }
        }
        dmc[idx] = m;
    }
};

// dm_cond over device shells: max |D_cart| over the block and over all density matrices
struct DmCondFn {
    const double* dj; int ndj; const double* dk; int ndk; double* dmc; int nsh, ncart; const int *sh_l, *sh_cart;
    B2_HD void operator()(long idx) const
    {
        int i = (int)(idx / nsh), j = (int)(idx - (long)i * nsh);
        int ni = (sh_l[i] + 1) * (sh_l[i] + 2) / 2, nj = (sh_l[j] + 1) * (sh_l[j] + 2) / 2;
        double m = 0.0;
        for (int pass = 0; pass < 2; pass++) {
            const double* D = pass ? dk : dj;
            int nd = pass ? ndk : ndj;
            if (!D) continue;
            for (int s = 0; s < nd; s++)
                for (int a = 0; a < ni; a++)
                    for (int b = 0; b < nj; b++) {
                        double v = fabs(D[(size_t)s * ncart * ncart + (size_t)(sh_cart[i] + a) * ncart + sh_cart[j] + b]);
                        m = v > m ? v : m;
                    }
        }
        dmc[idx] = m;
    }
};

// In-core J/K from stored integrals (CVHFnrs8_incore_drv, pyscf/lib/vhf/nr_incore.c:624; dot_eri_dm, pyscf/scf/hf.py:902-961):
// one thread per stored integral, every index permutation it stands for applied with reductions
//   J_kl += (ij|kl) D_ji ,  K_il += (ij|kl) D_jk        (pyscf/scf/hf.py:906-907)
// sym 8: eri[pq], p = i(i+1)/2+j >= q = k(k+1)/2+l;  sym 4: eri[p][q];  sym 1: eri[i][j][k][l].
struct IncoreJKFn {
    const double* eri; int sym, nao; long npair; const double* dm; int n_dm; double* vj; double* vk;
    static B2_HD void tri_decode(long t, long& a, long& b)   // t = a(a+1)/2 + b, a >= b
    {
        a = (long)((sqrt(8.0 * (double)t + 1.0) - 1.0) * 0.5);
        while (a * (a + 1) / 2 > t) a--;
        while ((a + 1) * (a + 2) / 2 <= t) a++;
        b = t - a * (a + 1) / 2;
    }
    B2_HD void one(double v, long i, long j, long k, long l) const
    {
        const long n = nao, n2 = n * n;
        for (int s = 0; s < n_dm; s++) {
            const double* D = dm + s * n2;
            if (vj) red_add(vj + s * n2 + k * n + l, v * D[j * n + i]);
            if (vk) red_add(vk + s * n2 + i * n + l, v * D[j * n + k]);
        }
    }
    B2_HD void operator()(long t) const
    {
        if (sym == 1) {
            const long n = nao;
            long l = t % n, r = t / n;
            long k = r % n; r /= n;
            long j = r % n, i = r / n;
            one(eri[t], i, j, k, l);
            return;
        }
        long p, q;
        if (sym == 8) tri_decode(t, p, q);
        else { p = t / npair; q = t - p * npair; }
        long i, j, k, l;
        tri_decode(p, i, j);
        tri_decode(q, k, l);
        double v = eri[t];
        if (v == 0.0) return;
        if (i == j) v *= 0.5;
        if (k == l) v *= 0.5;
        one(v, i, j, k, l); one(v, j, i, k, l); one(v, i, j, l, k); one(v, j, i, l, k);
        if (sym == 8) {
            if (p == q) return;      // (ij|kl) with ij == kl: the four bra/ket swaps above are all there is
            one(v, k, l, i, j); one(v, l, k, i, j); one(v, k, l, j, i); one(v, l, k, j, i);
        }
    }
};

inline int pair_class_id(int la, int lb) { return la * (la + 1) / 2 + lb; }

inline void set_err(b200jk_handle h, const std::string& m) { if (h) h->err = m; }

template <class T>
T* upload(const std::vector<T>& v)
{
    T* d = (T*)dev_alloc(v.size() * sizeof(T));
    if (!v.empty()) h2d(d, v.data(), v.size() * sizeof(T));
    return d;
}

}  // namespace b2host
