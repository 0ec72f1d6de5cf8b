// df_ao2mo.cuh — MO integral transforms of the density-fitting tensor (included by df.cu, which owns DFState).
//
//   b200jk_df_ao2mo       DF.ao2mo = get_mo_eri     pyscf/df/df.py:278-296  (_ao2mo.nr_e2 per row block + lib.dot)
//   b200jk_df_get_ao_eri  DF.get_eri = get_ao_eri   pyscf/df/df.py:269-276  (lib.dot(eri1.T, eri1) + ao2mo.restore(8))
//
// Stage 1, per block of local tensor rows P (device rows in place, host rows staged through d_stage on the copy stream):
//   Y[(P,nu), a]  = sum_mu B_P[nu,mu] Ca[mu,a]        straight from the packed rows (col_of of a pair-screened tensor)
//   L[P, ij]      = sum_nu Cb[nu,b] Y[(P,nu), a]      (a, b) = (i, j) or (j, i): the smaller coefficient set goes first
// with only i >= j kept (at i(i+1)/2 + j) for an s2 pair.  L of every local row, and L' of pair (3,4) unless it is pair (1,2),
// stay resident.
// Stage 2: out[ij, kl] = sum_P L[P, ij] L'[P, kl] in bands of output rows; each band is copied to the caller through pinned
// staging on the copy stream while the next band is computed.  With identical pairs the tiles above the diagonal of a band's
// diagonal block are skipped and mirrored on the device (one band: half of the output).  get_eri is stage 2 with L = L' = B,
// every band over all local rows by the same walk (host rows block by block, each block added).
//
// All three products run on ONE FP64 GEMM core on the tensor cores: DMMA.8x8x4 through nvcuda::wmma, CTA tile 64 x 64 x 16,
// four warps of 32 x 32, operands fetched into registers one k step ahead by element loaders (packed-symmetric rows, plain and
// transposed strided matrices) in one k loop, which DF-MP2's pair kernel and DF-RPA's Pi kernel run as well.  The emulation
// build runs the same CTA code, thread by thread and warp by warp, on a host model of the fragment operations.
// This file also holds what the four entry points on the tensor share: the call harness (MoCall), stage 1 (half_transform),
// the active-spin parser of DF-MP2 and DF-RPA and the one-CTA tree sum.
#include <thread>
#ifndef B200JK_EMULATE
#include <mma.h>
#endif

namespace ao2mo {

constexpr int BM = 64, BN = 64, BK = 16, NT = 128;
constexpr int LDA = BK + 4, LDB = BN + 4, LDC = BN + 4;     // padded shared rows; every fragment starts 32-byte aligned
constexpr int SM_AB = BM * LDA + BK * LDB, SM_C = BM * LDC;
constexpr int SMEM = SM_AB > SM_C ? SM_AB : SM_C;           // the C staging of the epilogue reuses the operand tiles
constexpr int PER_T = BM * BK / NT;                         // operand elements each thread stages per k step
static_assert(BM * BK == BK * BN && BM == 64 && BN == 64 && NT == 128, "four warps of 32 x 32");

#ifndef B200JK_EMULATE
#define AO_D __device__ __forceinline__
namespace fr {
using namespace nvcuda;
typedef wmma::fragment<wmma::matrix_a, 8, 8, 4, double, wmma::row_major> A;
typedef wmma::fragment<wmma::matrix_b, 8, 8, 4, double, wmma::row_major> B;
typedef wmma::fragment<wmma::accumulator, 8, 8, 4, double> C;
AO_D void zero(C& c) { wmma::fill_fragment(c, 0.0); }
AO_D void load(A& a, const double* p, int ld) { wmma::load_matrix_sync(a, p, ld); }
AO_D void load(B& b, const double* p, int ld) { wmma::load_matrix_sync(b, p, ld); }
AO_D void mma(C& c, const A& a, const B& b) { wmma::mma_sync(c, a, b, c); }
AO_D void store(double* p, const C& c, int ld) { wmma::store_matrix_sync(p, c, ld, wmma::mem_row_major); }
}  // namespace fr
#else
#define AO_D inline
// host model of the warp-wide 8x8x4 FP64 fragments: each holds the whole tile of its warp, row-major
namespace fr {
struct A { double x[8 * 4]; };
struct B { double x[4 * 8]; };
struct C { double x[8 * 8]; };
inline void zero(C& c) { for (double& v : c.x) v = 0.0; }
inline void load(A& a, const double* p, int ld) { for (int i = 0; i < 8; i++) for (int k = 0; k < 4; k++) a.x[i * 4 + k] = p[i * ld + k]; }
inline void load(B& b, const double* p, int ld) { for (int k = 0; k < 4; k++) for (int j = 0; j < 8; j++) b.x[k * 8 + j] = p[k * ld + j]; }
inline void mma(C& c, const A& a, const B& b)
{
    for (int i = 0; i < 8; i++)
        for (int j = 0; j < 8; j++) {
            double s = c.x[i * 8 + j];
            for (int k = 0; k < 4; k++) s += a.x[i * 4 + k] * b.x[k * 8 + j];
            c.x[i * 8 + j] = s;
        }
}
inline void store(double* p, const C& c, int ld) { for (int i = 0; i < 8; i++) for (int j = 0; j < 8; j++) p[i * ld + j] = c.x[i * 8 + j]; }
}  // namespace fr
#endif

// C[m, n] = sum_k a(m, k) b(k, n), m < M, n < N; st(m, n, value) writes one element.  A loader with MFAST (B: NFAST) is read
// with consecutive threads on consecutive m (n), else on consecutive k.  skip != 0: CTA tiles wholly above the diagonal (global
// row = row_off + m) and wholly left of column col_end are not computed (the caller mirrors them).
template <class LA, class LB, class ST>
struct Gemm {
    typedef LA TA; typedef LB TB;
    long M, N, K; LA a; LB b; ST st;
    int skip; long row_off, col_end;
};

template <class G>
AO_D bool skipped(const G& g, long m0, long n0)
{
    const long n_end = n0 + BN < g.N ? n0 + BN : g.N;
    return g.skip && n0 > g.row_off + m0 + BM - 1 && n_end <= g.col_end;
}
template <class G>
AO_D void tile_index_a(int e, int& m, int& k) { if (G::TA::MFAST) { m = e % BM; k = e / BM; } else { k = e % BK; m = e / BK; } }
template <class G>
AO_D void tile_index_b(int e, int& k, int& n) { if (G::TB::NFAST) { n = e % BN; k = e / BN; } else { k = e % BK; n = e / BK; } }

template <class G>
AO_D void fetch(const G& g, long m0, long n0, long k0, int t, double* ra, double* rb)
{
    for (int q = 0; q < PER_T; q++) {
        int m, n, k;
        tile_index_a<G>(t + q * NT, m, k);
        ra[q] = (m0 + m < g.M && k0 + k < g.K) ? g.a(m0 + m, k0 + k) : 0.0;
        tile_index_b<G>(t + q * NT, k, n);
        rb[q] = (n0 + n < g.N && k0 + k < g.K) ? g.b(k0 + k, n0 + n) : 0.0;
    }
}
template <class G>
AO_D void put(double* sm, int t, const double* ra, const double* rb)
{
    for (int q = 0; q < PER_T; q++) {
        int m, n, k;
        tile_index_a<G>(t + q * NT, m, k);
        sm[m * LDA + k] = ra[q];
        tile_index_b<G>(t + q * NT, k, n);
        sm[BM * LDA + k * LDB + n] = rb[q];
    }
}
AO_D void warp_mma(const double* sm, int w, fr::C (&c)[4][4])
{
    const int wm = (w >> 1) * 32, wn = (w & 1) * 32;
    for (int kk = 0; kk < BK; kk += 4) {
        fr::A a[4];
        fr::B b[4];
        for (int i = 0; i < 4; i++) fr::load(a[i], sm + (wm + 8 * i) * LDA + kk, LDA);
        for (int j = 0; j < 4; j++) fr::load(b[j], sm + BM * LDA + kk * LDB + wn + 8 * j, LDB);
        for (int i = 0; i < 4; i++)
            for (int j = 0; j < 4; j++) fr::mma(c[i][j], a[i], b[j]);
    }
}
AO_D void warp_store(double* sm, int w, const fr::C (&c)[4][4])
{
    const int wm = (w >> 1) * 32, wn = (w & 1) * 32;
    for (int i = 0; i < 4; i++)
        for (int j = 0; j < 4; j++) fr::store(sm + (wm + 8 * i) * LDC + wn + 8 * j, c[i][j], LDC);
}
template <class G>
AO_D void epilogue(const G& g, const double* sm, long m0, long n0, int t)
{
    for (int e = t; e < BM * BN; e += NT) {
        const int m = e / BN, n = e % BN;
        if (m0 + m < g.M && n0 + n < g.N) g.st(m0 + m, n0 + n, sm[m * LDC + n]);
    }
}

AO_D void red_step(double* red, int t, int s, int T) { if (t < s) { red[t] += red[t + s]; red[T + t] += red[T + t + s]; } }

// A-operand hook of the k loop: at(k0, t) when thread t fetches k step k0, apply(ra) to its A operand of that step at the put
struct NoHook {
    AO_D void at(long, int) {}
    AO_D void apply(double*) const {}
};

constexpr int RT = 256;     // threads of tree_sum

#ifndef B200JK_EMULATE
// One group of four warps (thread t of NT): c = sum over the k steps k0 = k_first, k_first + k_step, ... < k_end of the tile
// (m0, n0) of g (steps past g.K read zeros), the operands staged through sm.  Every thread of the CTA must run the same number
// of steps: each step has two barriers.
template <class G, class H>
AO_D void k_loop(const G& g, long m0, long n0, long k_first, long k_step, long k_end, double* sm, int t, H& hook,
                 fr::C (&c)[4][4])
{
#pragma unroll
    for (int i = 0; i < 4; i++)
#pragma unroll
        for (int j = 0; j < 4; j++) fr::zero(c[i][j]);
    double ra[PER_T], rb[PER_T];
    fetch(g, m0, n0, k_first, t, ra, rb);
    hook.at(k_first, t);
    for (long k0 = k_first; k0 < k_end; k0 += k_step) {
        hook.apply(ra);
        put<G>(sm, t, ra, rb);
        __syncthreads();
        if (k0 + k_step < k_end) {     // next k step in flight during the MMAs
            fetch(g, m0, n0, k0 + k_step, t, ra, rb);
            hook.at(k0 + k_step, t);
        }
        warp_mma(sm, t >> 5, c);
        __syncthreads();
    }
}

template <class G>
__global__ void __launch_bounds__(NT) f64gemm_kernel(G g, long n_base)
{
    __shared__ __align__(128) double sm[SMEM];
    const long m0 = (long)blockIdx.x * BM, n0 = n_base + (long)blockIdx.y * BN;
    if (skipped(g, m0, n0)) return;
    const int t = threadIdx.x;
    fr::C c[4][4];
    NoHook hk;
    k_loop(g, m0, n0, 0, BK, g.K, sm, t, hk, c);
    warp_store(sm, t >> 5, c);
    __syncthreads();
    epilogue(g, sm, m0, n0, t);
}

// one CTA of RT threads: out[0, 1] = the two sums over the shares share(t, a, b) of its threads, added in a fixed tree
template <class F>
__global__ void __launch_bounds__(RT) tree_sum_kernel(F share, double* out)
{
    __shared__ double red[2 * RT];
    const int t = threadIdx.x;
    double a = 0.0, b = 0.0;
    share(t, a, b);
    red[t] = a; red[RT + t] = b;
    __syncthreads();
    for (int s = RT / 2; s > 0; s >>= 1) {
        red_step(red, t, s, RT);
        __syncthreads();
    }
    if (t == 0) { out[0] = red[0]; out[1] = red[RT]; }
}
template <class F>
static void tree_sum(const F& share, double* out, cudaStream_t s)
{
    tree_sum_kernel<F><<<1, RT, 0, s>>>(share, out);
    CK(cudaGetLastError());
}
template <class G>
static void gemm(const G& g, cudaStream_t s)
{
    if (g.M <= 0 || g.N <= 0) return;
    const long gx = (g.M + BM - 1) / BM, gy = (g.N + BN - 1) / BN;
    if (gx > 0x7fffffffL) throw std::runtime_error("ao2mo: GEMM with too many rows");
    for (long y0 = 0; y0 < gy; y0 += 65535)
        f64gemm_kernel<G><<<dim3((unsigned)gx, (unsigned)std::min<long>(65535, gy - y0)), NT, 0, s>>>(g, y0 * BN);
    CK(cudaGetLastError());
}
#else
// the device k_loop, thread by thread and warp by warp on the host model of the fragments: c[w] of warp w, hook copied per thread
typedef fr::C Acc[4][4];
template <class G, class H>
static void k_loop(const G& g, long m0, long n0, long k_first, long k_step, long k_end, double* sm, const H& hook, Acc* c)
{
    std::vector<double> ra(NT * PER_T), rb(NT * PER_T);
    std::vector<H> hk(NT, hook);
    for (int w = 0; w < 4; w++)
        for (int i = 0; i < 4; i++)
            for (int j = 0; j < 4; j++) fr::zero(c[w][i][j]);
    for (int t = 0; t < NT; t++) {
        fetch(g, m0, n0, k_first, t, &ra[t * PER_T], &rb[t * PER_T]);
        hk[t].at(k_first, t);
    }
    for (long k0 = k_first; k0 < k_end; k0 += k_step) {
        for (int t = 0; t < NT; t++) {
            hk[t].apply(&ra[t * PER_T]);
            put<G>(sm, t, &ra[t * PER_T], &rb[t * PER_T]);
        }
        if (k0 + k_step < k_end)
            for (int t = 0; t < NT; t++) {
                fetch(g, m0, n0, k0 + k_step, t, &ra[t * PER_T], &rb[t * PER_T]);
                hk[t].at(k0 + k_step, t);
            }
        for (int w = 0; w < 4; w++) warp_mma(sm, w, c[w]);
    }
}

template <class G>
static void gemm(const G& g, stream_t)
{
    std::vector<double> sm(SMEM);
    Acc c[4];
    for (long m0 = 0; m0 < g.M; m0 += BM)
        for (long n0 = 0; n0 < g.N; n0 += BN) {
            if (skipped(g, m0, n0)) continue;
            k_loop(g, m0, n0, 0, BK, g.K, sm.data(), NoHook{}, c);
            for (int w = 0; w < 4; w++) warp_store(sm.data(), w, c[w]);
            for (int t = 0; t < NT; t++) epilogue(g, sm.data(), m0, n0, t);
        }
}

template <class F>
static void tree_sum(const F& share, double* out, stream_t)
{
    std::vector<double> red(2 * RT);
    for (int t = 0; t < RT; t++) {
        double a = 0.0, b = 0.0;
        share(t, a, b);
        red[t] = a; red[RT + t] = b;
    }
    for (int s = RT / 2; s > 0; s >>= 1)
        for (int t = 0; t < RT; t++) red_step(red.data(), t, s, RT);
    out[0] = red[0]; out[1] = red[RT];
}
#endif

// ---- operand loaders and stores ---------------------------------------------------------------------------------------
// a(m, k) = B_P[nu, k], m = P nao + nu: packed tensor rows (row P at rows + P ld), unpacked on the fly
struct TriRowsA {
    const double* rows; long ld; const int* col_of; int nao;
    static constexpr bool MFAST = false;
    B2_HD double operator()(long m, long k) const
    {
        const long P = m / nao, nu = m - P * nao;
        const long hi = nu >= k ? nu : k, lo = nu >= k ? k : nu;
        return packed_elem(rows + P * ld, col_of, hi * (hi + 1) / 2 + lo);
    }
};
// a(m, k) = p[k ld + m]
struct TransA {
    const double* p; long ld;
    static constexpr bool MFAST = true;
    B2_HD double operator()(long m, long k) const { return p[k * ld + m]; }
};
// b(k, n) = p[k ld + n]
struct RowsB {
    const double* p; long ld;
    static constexpr bool NFAST = true;
    B2_HD double operator()(long k, long n) const { return p[k * ld + n]; }
};
// b(k, n) = Y[(P nao + k) na + a], n = P na + a
struct YColsB {
    const double* y; int nao, na;
    static constexpr bool NFAST = true;
    B2_HD double operator()(long k, long n) const
    {
        const long P = n / na, a = n - P * na;
        return y[(P * nao + k) * na + a];
    }
};
// packed columns of tensor rows k: a(m, k) = B[k][c0 + m], b(k, n) = B[k][n] (packed pair indices, col_of when screened)
struct PackedColsA {
    const double* rows; long ld; const int* col_of; long c0;
    static constexpr bool MFAST = true;
    B2_HD double operator()(long m, long k) const { return packed_elem(rows + k * ld, col_of, c0 + m); }
};
struct PackedColsB {
    const double* rows; long ld; const int* col_of;
    static constexpr bool NFAST = true;
    B2_HD double operator()(long k, long n) const { return packed_elem(rows + k * ld, col_of, n); }
};
struct RowsSt {
    double* p; long ld;
    B2_HD void operator()(long m, long n, double v) const { p[m * ld + n] = v; }
};
// L[P][ij] from Z[b, (P, a)]: (i, j) = (b, a) when swap, else (a, b); s2 keeps i >= j at i(i+1)/2 + j, s1 puts (i, j) at i nj + j
struct LSt {
    double* L; long nij; int na, nj, swap, s2;
    B2_HD void operator()(long m, long n, double v) const
    {
        const long P = n / na, a = n - P * na;
        const long i = swap ? m : a, j = swap ? a : m;
        if (s2) { if (i >= j) L[P * nij + i * (i + 1) / 2 + j] = v; }
        else L[P * nij + i * nj + j] = v;
    }
};
// band of the s8 triangle, rows [r0, r0 + M): element (i, n <= i) at i(i+1)/2 + n - r0(r0+1)/2; acc: add (further row blocks)
struct TriBandSt {
    double* p; long r0; int acc;
    B2_HD void operator()(long m, long n, double v) const
    {
        const long i = r0 + m;
        if (n > i) return;
        double* q = p + i * (i + 1) / 2 + n - r0 * (r0 + 1) / 2;
        if (acc) *q += v; else *q = v;
    }
};
// rows [r0, r0 + nb) of a symmetric output held as a band buf[nb][ld]: the strict upper part of its diagonal block from the lower
struct MirrorBandFn {
    double* p; long ld, r0; long nb;
    B2_HD void operator()(long idx) const
    {
        const long m = idx / nb, c = idx - m * nb;
        if (c > m) p[m * ld + r0 + c] = p[c * ld + r0 + m];
    }
};

// host copy of a band into the caller's array, in up to 8 threads of >= 32 MiB (the first touch of a fresh numpy array and the
// copy out of pinned memory run at a few GB/s per core)
static void par_memcpy(void* dst, const void* src, size_t n)
{
    const size_t chunk = 32UL << 20;
    const int nt = (int)std::min<size_t>(8, std::max<size_t>(1, n / chunk));
    if (nt == 1) { memcpy(dst, src, n); return; }
    std::vector<std::thread> th;
    const size_t per = (n + nt - 1) / nt;
    for (int t = 0; t < nt; t++) {
        const size_t o = (size_t)t * per, len = o < n ? std::min(per, n - o) : 0;
        th.emplace_back([=]() { memcpy((char*)dst + o, (const char*)src + o, len); });
    }
    for (std::thread& x : th) x.join();
}

// Bands b = 0..nb-1 of the output: compute(b, dbuf) fills a device buffer on the compute stream and returns its bytes; the copy
// to a pinned buffer runs on the copy stream while band b + 1 is computed, and the host then hands it to sink(b, src, bytes),
// which moves it into the caller's array.  cap: bytes of the largest band.  ms2 accumulates the device time of compute().  The
// two pinned buffers stay on the handle (h_pin) for the next call: a CASSCF macro iteration calls ao2mo every time, and pinning
// hundreds of MB costs more than a small transform.
template <class FC, class FS>
static void band_pipeline(DFState* d, stream_t st, int nb, size_t cap, FC compute, FS sink, double& ms2)
{
    double* dbuf[2] = {(double*)dev_alloc(cap), nb > 1 ? (double*)dev_alloc(cap) : nullptr};
    size_t bytes[2] = {0, 0};
#ifndef B200JK_EMULATE
    const cudaStream_t cs = d->rows.copy_stream();
    if (d->pin_cap < cap) {
        for (double*& p : d->h_pin) { if (p) CK(cudaFreeHost(p)); p = nullptr; }
        d->pin_cap = 0;
        for (double*& p : d->h_pin) CK(cudaHostAlloc((void**)&p, cap, cudaHostAllocDefault));
        d->pin_cap = cap;
    }
    double* hbuf[2] = {d->h_pin[0], d->h_pin[1]};
    cudaEvent_t ev[8] = {};     // [0,1] band computed, [2,3] band copied, [4..7] compute start / end of the band in each slot
    for (int i = 0; i < 8; i++) CK(cudaEventCreateWithFlags(&ev[i], i < 4 ? cudaEventDisableTiming : cudaEventDefault));
    try {
        auto drain = [&](int b) {       // band b's copy is done: time its compute, move it to the caller
            const int s = b & 1;
            CK(cudaEventSynchronize(ev[2 + s]));
            float t = 0;
            CK(cudaEventElapsedTime(&t, ev[4 + 2 * s], ev[5 + 2 * s]));
            ms2 += t;
            sink(b, hbuf[s], bytes[s]);
        };
        for (int b = 0; b < nb; b++) {
            const int s = b & 1;
            if (b >= 2) drain(b - 2);                            // frees hbuf[s]; dbuf[s] was read by that copy
            CK(cudaEventRecord(ev[4 + 2 * s], st));
            bytes[s] = compute(b, dbuf[s]);
            CK(cudaEventRecord(ev[5 + 2 * s], st));
            CK(cudaEventRecord(ev[s], st));
            CK(cudaStreamWaitEvent(cs, ev[s], 0));
            CK(cudaMemcpyAsync(hbuf[s], dbuf[s], bytes[s], cudaMemcpyDeviceToHost, cs));
            CK(cudaEventRecord(ev[2 + s], cs));
            if (b + 1 < nb) CK(cudaStreamWaitEvent(st, ev[2 + (s ^ 1)], 0));   // the next band overwrites the other buffer
        }
        for (int b = std::max(0, nb - 2); b < nb; b++) drain(b);
    } catch (...) {
        cudaDeviceSynchronize();
        for (cudaEvent_t e : ev) cudaEventDestroy(e);
        dev_free(dbuf[0]); dev_free(dbuf[1]);
        throw;
    }
    for (cudaEvent_t e : ev) cudaEventDestroy(e);
#else
    (void)d; (void)st; (void)ms2;
    for (int b = 0; b < nb; b++) {
        bytes[b & 1] = compute(b, dbuf[b & 1]);
        sink(b, dbuf[b & 1], bytes[b & 1]);
    }
#endif
    dev_free(dbuf[0]); dev_free(dbuf[1]);
}

}  // namespace ao2mo

// largest band of output rows: at most 256 MiB (or the test cap of b200jk_df_set_ao2mo_tile) per band
static long ao2mo_band_rows(const DFState* d, long nrows, long row_bytes)
{
    long r = std::max(1L, std::min(nrows, (256L << 20) / std::max(1L, row_bytes)));
    if (d->ao2mo_tile_rows > 0) r = std::min<long>(r, d->ao2mo_tile_rows);
    return r;
}

static void ao2mo_check_fit(double need, const char* what)
{
#ifndef B200JK_EMULATE
    size_t freeb = 0, totb = 0;
    CK(cudaMemGetInfo(&freeb, &totb));
    if (need > 0.95 * (double)freeb) {
        char buf[400];
        snprintf(buf, sizeof buf, "%s need %.2f GB of device memory next to the DF tensor, but only %.2f GB are free; "
                 "use fewer orbitals per call", what, need / 1e9, freeb / 1e9);
        throw std::runtime_error(buf);
    }
#else
    (void)need; (void)what;
#endif
}

// One call of an entry point that reads the resident tensor (ao2mo, get_ao_eri, DF-MP2, DF-RPA).  The constructor checks that
// the tensor is built and not sharded (why: the caller's reason), selects the device and stream and starts the host clock.
// finish() synchronises with a check, so that an asynchronous fault is reported, frees the buffers and returns the host ms;
// the destructor frees what is still owned after an unchecked synchronisation, so that an error path cannot throw again.
struct MoCall {
    DFState* d;
    stream_t st = 0;
    std::vector<void*> owned;
    std::chrono::steady_clock::time_point t0;

    MoCall(b200jk_handle h, const char* fn, const char* why = "") : d(h->df)
    {
        if (!d || !d->d_cderi) throw std::runtime_error(std::string("call b200jk_df_build (or b200jk_df_set_cderi) before ") + fn);
        if (d->build_world != 1) throw std::runtime_error(std::string(fn) + ": a sharded tensor is not supported" + why);
#ifndef B200JK_EMULATE
        CK(cudaSetDevice(h->device));
        st = h->stream;
#endif
        t0 = std::chrono::steady_clock::now();
    }
    ~MoCall()
    {
#ifndef B200JK_EMULATE
        cudaDeviceSynchronize();
#endif
        for (void* p : owned) dev_free(p);
    }
    void* alloc(size_t bytes)
    {
        void* p = dev_alloc(bytes);
        owned.push_back(p);
        return p;
    }
    void free(void* p)
    {
        dev_sync();
        owned.erase(std::find(owned.begin(), owned.end(), p));
        dev_free(p);
    }
    double finish()
    {
        dev_sync();
        for (void* p : owned) dev_free(p);
        owned.clear();
        return std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now() - t0).count();
    }
};

// n stage times of the last call, from the DFState array src of N, into ms (zeros past N)
template <int N>
static int mo_times(b200jk_handle h, double (DFState::*src)[N], double* ms, int n)
{
    if (!h || !h->df || !ms) { set_err(h, "call b200jk_df_build first"); return 1; }
    for (int i = 0; i < n; i++) ms[i] = i < N ? (h->df->*src)[i] : 0.0;
    return 0;
}

// One coefficient pair of stage 1: host sets c[0] [nao][n[0]] and c[1] [nao][n[1]], their device copies dc, and the output
// L[P][nij] (s2: i >= j at i(i+1)/2 + j, else i n[1] + j) over the local rows P.
struct HalfPair { const double* c[2]; int n[2]; int s2; long nij; double* L; double* dc[2]; };

// The spins of an occupied / virtual calculation (DF-MP2, DF-RPA) with orbitals on both sides: their stage-1 pairs (C_occ,
// C_vir) in spin order, pr_of[s] = index in pr (-1: inactive) and the largest set contracted first.  e0, e1: the per-spin
// arrays the caller needs of an active spin.
struct ActiveSpins {
    HalfPair pr[2];
    int npr = 0, pr_of[2] = {-1, -1}, na_max = 1;
    ActiveSpins(int nspin, const double* const* c_occ, const int* nocc, const double* const* c_vir, const int* nvir,
                const double* const* e0, const double* const* e1)
    {
        for (int s = 0; s < nspin; s++) {
            if (nocc[s] < 0 || nvir[s] < 0) throw std::runtime_error("bad arguments: negative orbital count");
            if (nocc[s] == 0 || nvir[s] == 0) continue;
            if (!c_occ[s] || !c_vir[s] || !e0[s] || !e1[s]) throw std::runtime_error("bad arguments");
            pr[npr] = HalfPair{{c_occ[s], c_vir[s]}, {nocc[s], nvir[s]}, 0, (long)nocc[s] * nvir[s], nullptr, {nullptr, nullptr}};
            na_max = std::max(na_max, std::min(nocc[s], nvir[s]));
            pr_of[s] = npr++;
        }
    }
    bool active(int s) const { return pr_of[s] >= 0; }
};

// tensor rows per stage-1 block: Y of a block at most 512 MiB; na_max = largest set contracted first
static int half_block_rows(int nrow, int nao, int na_max)
{
    return (int)std::max<long>(1, std::min<long>(std::max(nrow, 1), (512L << 20) / ((long)nao * na_max * 8)));
}

// Stage 1 on the compute stream: allocates L and the device coefficients of every pair in pr[0, npr) through the call,
// uploads the coefficients and fills L from all local rows (device rows in place, host rows through the staging buffers), in
// blocks of rb rows through a temporary Y [rb][nao][na_max] that is freed again.  Returns the device ms of the GEMMs.
static double half_transform(MoCall& c, int nao, HalfPair* pr, int npr, int rb, int na_max)
{
    if (npr == 0) return 0.0;
    DFState* d = c.d;
    const stream_t st = c.st;
    const long ld = d->ncol;
    const int* col_of = d->d_col_of;
    for (int q = 0; q < npr; q++) {
        pr[q].L = (double*)c.alloc((size_t)std::max(d->nrow, 1) * pr[q].nij * 8);
        for (int s = 0; s < 2; s++) {
            pr[q].dc[s] = (double*)c.alloc((size_t)nao * pr[q].n[s] * 8);
            h2d(pr[q].dc[s], pr[q].c[s], (size_t)nao * pr[q].n[s] * 8, st);
        }
    }
    double* d_Y = (double*)c.alloc((size_t)rb * nao * na_max * 8);
    StageTimer tm;
    // ---- stage 1 on the rows [r0, r0 + nr) at src
    auto half = [&](const double* src, int r0, int nr) {
        tm.mark(0, st);
        for (int q = 0; q < npr; q++) {
            HalfPair& p = pr[q];
            const int f = p.n[0] <= p.n[1] ? 0 : 1;     // the smaller set is contracted first
            const int na = p.n[f], nb_ = p.n[1 - f];
            ao2mo::Gemm<ao2mo::TriRowsA, ao2mo::RowsB, ao2mo::RowsSt> g1{(long)nr * nao, na, nao, {src, ld, col_of, nao},
                                                                          {p.dc[f], na}, {d_Y, na}, 0, 0, 0};
            ao2mo::gemm(g1, st);
            ao2mo::Gemm<ao2mo::TransA, ao2mo::YColsB, ao2mo::LSt> g2{nb_, (long)nr * na, nao, {p.dc[1 - f], nb_}, {d_Y, nao, na},
                                                                     {p.L + (size_t)r0 * p.nij, p.nij, na, p.n[1], f == 1, p.s2}, 0, 0, 0};
            ao2mo::gemm(g2, st);
        }
        tm.mark(-1, st);
    };
    d->rows.walk(d->d_cderi, 0, d->nrow, std::min(rb, d->rows.stage_rows), false, st, [&](const double* src, int r0, int nr) {
        for (int q = 0; q < nr; q += rb) half(src + (size_t)q * ld, r0 + q, std::min(rb, nr - q));
    });
    c.free(d_Y);
    double ms = 0.0;
    tm.read(&ms, nullptr, 1);
    return ms;
}

extern "C" int b200jk_df_ao2mo(b200jk_handle h, const double* c1, int n1, const double* c2, int n2, int s2_12, const double* c3,
                               int n3, const double* c4, int n4, int s2_34, double* out)
{
    if (!h) return 1;
    try {
        MoCall c(h, "b200jk_df_ao2mo");
        DFState* d = c.d;
        const bool same = c3 == nullptr;
        if (same) { c3 = c1; n3 = n1; c4 = c2; n4 = n2; s2_34 = s2_12; }
        if (!c1 || !c2 || !c4 || !out || n1 < 1 || n2 < 1 || n3 < 1 || n4 < 1) throw std::runtime_error("bad arguments");
        if ((s2_12 && n1 != n2) || (s2_34 && n3 != n4)) throw std::runtime_error("an s2 pair needs two sets of equal size");
        const int nao = h->nsph, nrow = d->nrow;
        HalfPair pr[2] = {{{c1, c2}, {n1, n2}, s2_12, 0, nullptr, {nullptr, nullptr}},
                          {{c3, c4}, {n3, n4}, s2_34, 0, nullptr, {nullptr, nullptr}}};
        const int npr = same ? 1 : 2;
        int na_max = 1;
        for (HalfPair& p : pr) {
            p.nij = p.s2 ? (long)p.n[0] * (p.n[0] + 1) / 2 : (long)p.n[0] * p.n[1];
            na_max = std::max(na_max, std::min(p.n[0], p.n[1]));
        }
        const long nij = pr[0].nij, nkl = pr[npr - 1].nij;
        const int rb = half_block_rows(nrow, nao, na_max);
        const long band = ao2mo_band_rows(d, nij, nkl * 8);
        ao2mo_check_fit(8.0 * ((double)nrow * (nij + (same ? 0 : nkl)) + (double)rb * nao * na_max + 2.0 * band * nkl),
                        "the half-transformed integrals L[naux, nij] (and L[naux, nkl]) with their work buffers");
        const double ms1 = half_transform(c, nao, pr, npr, rb, na_max);
        double ms2 = 0.0;
        // ---- stage 2: bands of output rows [r0, r1)
        const double* Lij = pr[0].L;
        const double* Lkl = pr[npr - 1].L;
        const int nbands = (int)((nij + band - 1) / band);
        ao2mo::band_pipeline(d, c.st, nbands, (size_t)band * nkl * 8, [&](int b, double* buf) -> size_t {
            const long r0 = (long)b * band, r1 = std::min(nij, r0 + band);
            ao2mo::Gemm<ao2mo::TransA, ao2mo::RowsB, ao2mo::RowsSt> g{r1 - r0, nkl, nrow, {Lij + r0, nij}, {Lkl, nkl}, {buf, nkl},
                                                                      same ? 1 : 0, r0, r1};
            ao2mo::gemm(g, c.st);
            if (same) { ao2mo::MirrorBandFn mf{buf, nkl, r0, r1 - r0}; launch_1d((r1 - r0) * (r1 - r0), mf, c.st); }
            return (size_t)(r1 - r0) * nkl * 8;
        }, [&](int b, const void* src, size_t n) { ao2mo::par_memcpy(out + (size_t)b * band * nkl, src, n); }, ms2);
        d->ao2mo_ms[0] = ms1; d->ao2mo_ms[1] = ms2;
        d->ao2mo_ms[2] = c.finish();
    } catch (std::exception& e) { set_err(h, e.what()); return 2; }
    return 0;
}

extern "C" int b200jk_df_get_ao_eri(b200jk_handle h, double* out)
{
    if (!h) return 1;
    try {
        MoCall c(h, "b200jk_df_get_ao_eri");
        DFState* d = c.d;
        if (!out) throw std::runtime_error("bad arguments");
        const long npair = d->npair, ld = d->ncol;
        const int* col_of = d->d_col_of;
        // bands of s8 rows [r0, r1), each at most the bytes of ao2mo_band_rows(npair rows of npair columns)
        const long band = ao2mo_band_rows(d, npair, npair * 8);
        std::vector<long> rows{0};
        while (rows.back() < npair) {
            const long r0 = rows.back();
            long r1 = r0 + 1;
            while (r1 < npair && r1 - r0 < band && (r1 + 1) * (r1 + 2) / 2 - r0 * (r0 + 1) / 2 <= band * npair) r1++;
            rows.push_back(r1);
        }
        ao2mo_check_fit(16.0 * band * npair, "the output bands of get_ao_eri");
        double ms2 = 0.0;
        ao2mo::band_pipeline(d, c.st, (int)rows.size() - 1, (size_t)band * npair * 8, [&](int b, double* buf) -> size_t {
            const long r0 = rows[b], r1 = rows[b + 1];
            // every local row block adds to the band; the first one (device rows, or the first host block) stores
            d->rows.walk(d->d_cderi, 0, d->nrow, d->rows.stage_rows, false, c.st, [&](const double* src, int a0, int nr) {
                ao2mo::Gemm<ao2mo::PackedColsA, ao2mo::PackedColsB, ao2mo::TriBandSt> g{r1 - r0, r1, nr, {src, ld, col_of, r0},
                                                                                        {src, ld, col_of}, {buf, r0, a0 > 0}, 1, r0, r1};
                ao2mo::gemm(g, c.st);
            });
            return (size_t)(r1 * (r1 + 1) / 2 - r0 * (r0 + 1) / 2) * 8;
        }, [&](int b, const void* src, size_t n) { ao2mo::par_memcpy(out + rows[b] * (rows[b] + 1) / 2, src, n); }, ms2);
        d->ao2mo_ms[0] = 0.0; d->ao2mo_ms[1] = ms2;
        d->ao2mo_ms[2] = c.finish();
    } catch (std::exception& e) { set_err(h, e.what()); return 2; }
    return 0;
}

extern "C" int b200jk_df_set_ao2mo_tile(b200jk_handle h, int max_rows)
{
    if (!h || !h->df) { set_err(h, "call b200jk_df_build first"); return 1; }
    if (max_rows == 0 || max_rows < -1) { set_err(h, "bad output band cap"); return 1; }
    h->df->ao2mo_tile_rows = max_rows;
    return 0;
}

extern "C" int b200jk_df_ao2mo_times(b200jk_handle h, double* ms, int n) { return mo_times(h, &DFState::ao2mo_ms, ms, n); }
