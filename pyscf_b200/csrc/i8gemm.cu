// i8gemm.cu — host side of the int8-slice tensor-core GEMM (see i8gemm.cuh) + a C-ABI self-test entry.
#include "host_common.hpp"
#ifndef B200JK_EMULATE
#include <cudaTypedefs.h>
#include "i8gemm.cuh"
#include "i8gemm_host.hpp"

namespace b200jk {
namespace i8g {

static PFN_cuTensorMapEncodeTiled_v12000 get_encode()
{
    static PFN_cuTensorMapEncodeTiled_v12000 fn = nullptr;
    if (!fn) {
        cudaDriverEntryPointQueryResult qres;
        void* p = nullptr;
        CK(cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &qres));
        if (!p || qres != cudaDriverEntryPointSuccess) throw std::runtime_error("cuTensorMapEncodeTiled not available");
        fn = (PFN_cuTensorMapEncodeTiled_v12000)p;
    }
    return fn;
}

static void make_tmap(CUtensorMap* m, const void* base, uint64_t rows, uint64_t kp, uint32_t box_rows)
{
    cuuint64_t dims[2] = {kp, rows};
    cuuint64_t strides[1] = {kp};
    cuuint32_t box[2] = {(cuuint32_t)BK, box_rows};
    cuuint32_t estr[2] = {1, 1};
    CUresult r = get_encode()(m, CU_TENSOR_MAP_DATA_TYPE_UINT8, 2, const_cast<void*>(base), dims, strides, box, estr,
                              CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                              CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    if (r != CUDA_SUCCESS) throw std::runtime_error("cuTensorMapEncodeTiled failed: " + std::to_string((int)r));
}

void SliceStack::alloc(int rows, int k, int ns_)
{
    if (rows != R || k != K || ns_ != ns) zeroed_for = 0;
    R = rows; K = k; ns = ns_;
    Rp = ((rows + 255) / 256) * 256;   // multiple of both BM and BN
    Kp = ((k + BK - 1) / BK) * BK;
    size_t need = (size_t)ns * Rp * Kp;
    if (need > cap) { dev_free(q); q = (int8_t*)dev_alloc(need); cap = need; }
    if (Rp > ecap) { dev_free(E); E = (int*)dev_alloc((size_t)Rp * 4); ecap = Rp; }
    if (!maxbits_cap || (size_t)Rp > maxbits_cap) { dev_free(maxbits); maxbits = (unsigned long long*)dev_alloc((size_t)Rp * 8); maxbits_cap = Rp; }
}
void SliceStack::release() { dev_free(q); dev_free(E); dev_free(maxbits); q = nullptr; E = nullptr; maxbits = nullptr; cap = 0; ecap = 0; maxbits_cap = 0; }

// rows [row0, row0+rows) of an already allocated stack (S.alloc(total_rows, k, ns) + zero fill done by the caller)
void split_rows_into(SliceStack& S, int row0, const double* X, long ldx, int rows, cudaStream_t st)
{
    split_rows_kernel<<<(rows + 7) / 8, 256, 0, st>>>(X, ldx, rows, S.K, S.Rp, S.Kp, S.ns, row0, S.q, S.E);
    CK(cudaGetLastError());
}

// first half of split_rows for a matrix that is still being produced: allocation + cleared row maxima, which the producer
// (stage 1 of DF-K, GemmParams::rowmax) fills; split_rows_premax then cuts the slices without a row-maximum pass
void split_rows_prepare(SliceStack& S, int rows, int k, int ns, cudaStream_t st)
{
    S.alloc(rows, k, ns);
    S.zeroed_for = 0;
    S.dmax = 64;
    CK(cudaMemsetAsync(S.maxbits, 0, (size_t)rows * 8, st));
}
void split_rows_premax(SliceStack& S, const double* X, long ldx, int rows, int k, int ns, cudaStream_t st)
{
    if (S.R != rows || S.K != k || S.ns != ns) throw std::runtime_error("split_rows_premax: call split_rows_prepare first");
    if (S.Rp > rows) {
        for (int s = 0; s < ns; s++)
            CK(cudaMemsetAsync(S.q + ((size_t)s * S.Rp + rows) * S.Kp, 0, (size_t)(S.Rp - rows) * S.Kp, st));
        CK(cudaMemsetAsync(S.E + rows, 0, (size_t)(S.Rp - rows) * 4, st));
    }
    const long seglen = 8192;
    unsigned nseg = (unsigned)((S.Kp + seglen - 1) / seglen);
    split_long_kernel<<<dim3(nseg, rows), 256, 0, st>>>(X, ldx, k, S.Rp, S.Kp, ns, seglen, S.maxbits, S.q, S.E);
    CK(cudaGetLastError());
}

void split_rows(SliceStack& S, const double* X, long ldx, int rows, int k, int ns, cudaStream_t st)
{
    S.alloc(rows, k, ns);
    S.zeroed_for = 0;
    S.dmax = 64;
    if (S.Rp > rows) {   // zero the pad rows of every slice
        for (int s = 0; s < ns; s++)
            CK(cudaMemsetAsync(S.q + ((size_t)s * S.Rp + rows) * S.Kp, 0, (size_t)(S.Rp - rows) * S.Kp, st));
        CK(cudaMemsetAsync(S.E + rows, 0, (size_t)(S.Rp - rows) * 4, st));
    }
    if ((long)k >= 8192 && rows < 4096) {
        const long seglen = 8192;
        unsigned nseg = (unsigned)((S.Kp + seglen - 1) / seglen);
        CK(cudaMemsetAsync(S.maxbits, 0, (size_t)rows * 8, st));
        rowmax_kernel<<<dim3(nseg, rows), 256, 0, st>>>(X, ldx, k, seglen, S.maxbits);
        split_long_kernel<<<dim3(nseg, rows), 256, 0, st>>>(X, ldx, k, S.Rp, S.Kp, ns, seglen, S.maxbits, S.q, S.E);
    } else {
        split_rows_kernel<<<(rows + 7) / 8, 256, 0, st>>>(X, ldx, rows, k, S.Rp, S.Kp, ns, 0, S.q, S.E);
    }
    CK(cudaGetLastError());
}

// ---- the DF tensor from its packed rows (see i8gemm.cuh (3)) ----
// rowexp[nr][nao]: exponent of every row (P, a) of the unpacked tensor; cderi points at the first of the nr packed rows
void packed_rowexp(const double* cderi, long npair, int nao, int nr, int* rowexp, float* rownorm2, cudaStream_t st, const int* col_of)
{
    CK(cudaMemsetAsync(rowexp, 0x80, (size_t)nr * nao * 4, st));     // EXP_NONE
    if (rownorm2) CK(cudaMemsetAsync(rownorm2, 0, (size_t)nr * nao * 4, st));
    static bool configured = false;
    if (!configured) {
        CK(cudaFuncSetAttribute(packed_rowexp_kernel<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, 160 * 1024));
        CK(cudaFuncSetAttribute(packed_rowexp_kernel<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, 160 * 1024));
        configured = true;
    }
    if ((size_t)nao * 8 > 160 * 1024) throw std::runtime_error("packed_rowexp: nao too large for the shared-memory tables");
    for (int p0 = 0; p0 < nr; p0 += 32768) {
        int n = std::min(32768, nr - p0);
        const dim3 grid((nao + 63) / 64, n);
        if (col_of)
            packed_rowexp_kernel<true><<<grid, 256, (size_t)nao * 8, st>>>(cderi + (size_t)p0 * npair, npair, nao, rowexp + (size_t)p0 * nao,
                                                                           rownorm2 ? rownorm2 + (size_t)p0 * nao : nullptr, col_of);
        else
            packed_rowexp_kernel<false><<<grid, 256, (size_t)nao * 8, st>>>(cderi + (size_t)p0 * npair, npair, nao, rowexp + (size_t)p0 * nao,
                                                                            rownorm2 ? rownorm2 + (size_t)p0 * nao : nullptr, nullptr);
    }
    CK(cudaGetLastError());
}
// ---- stage 1 cutting the slices of Y itself (GemmParams::yq) ----
// cmax2[0] = max_i ||row i of X||^2 (X = the right factor of stage 1 as rows [ncol][k])
void colnorm_max(const double* X, long ldx, int nrows, int k, double* cmax2, cudaStream_t st)
{
    CK(cudaMemsetAsync(cmax2, 0, 8, st));
    colnorm_max_kernel<<<(nrows + 7) / 8, 256, 0, st>>>(X, ldx, nrows, k, reinterpret_cast<unsigned long long*>(cmax2));
    CK(cudaGetLastError());
}
// the Y stack of one block: rows = nao, columns (P, i) with i padded to a multiple of 16; pads are zeroed when the shape changes
// (the epilogue of stage 1 overwrites every real element of every block), exponents = the Cauchy-Schwarz bound of each row
void y_prepare(SliceStack& S, int nao, int nr, int ncolp, int ns, const float* rownorm2_block, const double* cmax2, cudaStream_t st)
{
    const int k = nr * ncolp;
    S.alloc(nao, k, ns);
    S.dmax = 64;
    const bool same = (S.zeroed_for == (long)nao * 1000003L + k);
    if (!same) {
        CK(cudaMemsetAsync(S.q, 0, (size_t)ns * S.Rp * S.Kp, st));
        CK(cudaMemsetAsync(S.E, 0, (size_t)S.Rp * 4, st));
        S.zeroed_for = (long)nao * 1000003L + k;
    }
    yexp_bound_kernel<<<(nao + 255) / 256, 256, 0, st>>>(rownorm2_block, nr, nao, cmax2, S.E);
    CK(cudaGetLastError());
}
// slices of the unpacked rows (P, a), P in [0, nr), into the rows out_row0 + P nao + a of an allocated stack
void split_packed_into(SliceStack& S, int out_row0, const double* cderi, long npair, int nao, int nr, const int* rowexp, cudaStream_t st,
                       const int* col_of)
{
    if (S.K != nao) throw std::runtime_error("split_packed: stack width does not match nao");
    S.dmax = S.ns <= 7 ? 127 : 64;
    const unsigned nt = (unsigned)(S.Kp / PT);
    for (int p0 = 0; p0 < nr; p0 += 32768) {
        int n = std::min(32768, nr - p0);
        const dim3 grid(nt, nt, n);
        const double* src = cderi + (size_t)p0 * npair;
        const int* ex = rowexp + (size_t)p0 * nao;
        if (S.ns == 7) {
            if (col_of) split_packed_kernel<true, true><<<grid, 256, 0, st>>>(src, npair, nao, ex, S.ns, S.Rp, S.Kp, out_row0 + p0 * nao, S.q, S.E, col_of);
            else split_packed_kernel<true, false><<<grid, 256, 0, st>>>(src, npair, nao, ex, S.ns, S.Rp, S.Kp, out_row0 + p0 * nao, S.q, S.E, nullptr);
        } else {
            if (col_of) split_packed_kernel<false, true><<<grid, 256, 0, st>>>(src, npair, nao, ex, S.ns, S.Rp, S.Kp, out_row0 + p0 * nao, S.q, S.E, col_of);
            else split_packed_kernel<false, false><<<grid, 256, 0, st>>>(src, npair, nao, ex, S.ns, S.Rp, S.Kp, out_row0 + p0 * nao, S.q, S.E, nullptr);
        }
    }
    CK(cudaGetLastError());
}
// a stack holding exactly these nr packed rows (allocated here, pad rows zeroed)
void split_packed(SliceStack& S, const double* cderi, long npair, int nao, int nr, const int* rowexp, int ns, cudaStream_t st, const int* col_of)
{
    const int rows = nr * nao;
    S.alloc(rows, nao, ns);
    if (S.Rp > rows) {
        for (int s = 0; s < ns; s++)
            CK(cudaMemsetAsync(S.q + ((size_t)s * S.Rp + rows) * S.Kp, 0, (size_t)(S.Rp - rows) * S.Kp, st));
        CK(cudaMemsetAsync(S.E + rows, 0, (size_t)(S.Rp - rows) * 4, st));
    }
    split_packed_into(S, 0, cderi, npair, nao, nr, rowexp, st, col_of);
}

static int sm_count()
{
    static int nsm = 0;
    if (!nsm) {
        int dev = 0;
        CK(cudaGetDevice(&dev));
        CK(cudaDeviceGetAttribute(&nsm, cudaDevAttrMultiProcessorCount, dev));
    }
    return nsm;
}

template <int NS>
static void launch_ns(unsigned grid, const CUtensorMap& ta, const CUtensorMap& tb, const GemmParams& P, cudaStream_t st)
{
    static bool configured = false;
    if (!configured) {
        CK(cudaFuncSetAttribute(i8gemm_kernel<NS>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem_bytes(NS)));
        configured = true;
    }
    i8gemm_kernel<NS><<<grid, NTHREADS, smem_bytes(NS), st>>>(ta, tb, P);
}
// the slice count is a template parameter of the kernel: the accumulators of all slice-pair groups live in registers
static void launch(unsigned grid, const CUtensorMap& ta, const CUtensorMap& tb, const GemmParams& P, cudaStream_t st)
{
    switch (P.ns) {
    case 1: launch_ns<1>(grid, ta, tb, P, st); break;
    case 2: launch_ns<2>(grid, ta, tb, P, st); break;
    case 3: launch_ns<3>(grid, ta, tb, P, st); break;
    case 4: launch_ns<4>(grid, ta, tb, P, st); break;
    case 5: launch_ns<5>(grid, ta, tb, P, st); break;
    case 6: launch_ns<6>(grid, ta, tb, P, st); break;
    case 7: launch_ns<7>(grid, ta, tb, P, st); break;
    case 8: launch_ns<8>(grid, ta, tb, P, st); break;
    default: throw std::runtime_error("i8gemm: slice count out of range");
    }
    CK(cudaGetLastError());
}

// Longest K range (in K blocks) whose slice-pair group sums are exact in int32: group ns-1 adds ns pairs of kr products of at
// most dmax_A dmax_B each, so ns kr dmax_A dmax_B <= 2^31 - 1.  Columns at or past the shorter operand's K are zero and count
// for nothing.  Returns the number of K blocks of the whole product when it fits in one range.
static int int32_kblocks(const SliceStack& A, const SliceStack& B)
{
    const long kmax = ((1L << 31) - 1) / ((long)A.ns * A.dmax * B.dmax);
    if (std::min(A.K, B.K) <= kmax) return A.Kp / BK;
    return (int)(kmax / BK);
}

// stage-1 GEMM of DF-K: rows [a_row0, a_row0+M) of A times B^T, one work item per tile, persistent grid
void gemm_ar(const SliceStack& A, int a_row0, int M, const SliceStack& B, double* C, long ldc, int inner, cudaStream_t st,
             unsigned long long* rowmax, const SliceStack* Yout, int y_ncolp)
{
    if (A.Kp != B.Kp || A.ns != B.ns) throw std::runtime_error("i8gemm_ar: operand stacks disagree");
    if (A.ns < 1 || A.ns > MAXS) throw std::runtime_error("i8gemm_ar: slice count out of range");
    if (a_row0 < 0 || M < 0 || a_row0 + M > A.R) throw std::runtime_error("i8gemm_ar: row block outside the A stack");
    if (int32_kblocks(A, B) < A.Kp / BK) throw std::runtime_error("i8gemm_ar: K too long for exact int32 slice-pair sums");
    const int nsm = sm_count();
    CUtensorMap ta, tb;
    make_tmap(&ta, A.q, (uint64_t)A.ns * A.Rp, A.Kp, BM);
    make_tmap(&tb, B.q, (uint64_t)B.ns * B.Rp, B.Kp, BN);
    GemmParams P{};
    P.M = M; P.N = B.R; P.Kp = A.Kp; P.Mp = A.Rp; P.Np = B.Rp; P.ns = A.ns; P.symmetric = 0;
    P.Ea = A.E; P.Eb = B.E; P.C = C; P.ldc = ldc; P.inner = inner; P.a_row0 = a_row0;
    const int ntiles = ((B.R + BN - 1) / BN) * ((M + BM - 1) / BM);
    P.ntiles = ntiles; P.ksplit = 1; P.kb_per = A.Kp / BK; P.accumulate = 0; P.rowmax = rowmax;
    if (Yout) {
        if (inner <= 0 || (y_ncolp & 15) || y_ncolp < B.R || (long)((M + inner - 1) / inner) * y_ncolp > Yout->Kp || Yout->R != inner)
            throw std::runtime_error("i8gemm_ar: inconsistent Y stack");
        P.yq = Yout->q; P.Ey = Yout->E; P.y_Rp = Yout->Rp; P.y_Kp = Yout->Kp; P.y_ncolp = y_ncolp;
    }
    launch((unsigned)std::min(ntiles, nsm), ta, tb, P, st);
}

// C += A B^T (upper triangle only when symmetric): stage 2 of DF-K.  Work items = tiles x K ranges, sized to fill whole
// waves of the persistent grid.
void gemm_ar_acc(const SliceStack& A, const SliceStack& B, double* C, long ldc, bool symmetric, cudaStream_t st, int kb_per)
{
    if (A.Kp != B.Kp || A.ns != B.ns) throw std::runtime_error("i8gemm_ar_acc: operand stacks disagree");
    if (A.ns < 1 || A.ns > MAXS) throw std::runtime_error("i8gemm_ar_acc: slice count out of range");
    const int nsm = sm_count();
    CUtensorMap ta, tb;
    make_tmap(&ta, A.q, (uint64_t)A.ns * A.Rp, A.Kp, BM);
    make_tmap(&tb, B.q, (uint64_t)B.ns * B.Rp, B.Kp, BN);
    GemmParams P{};
    P.M = A.R; P.N = B.R; P.Kp = A.Kp; P.Mp = A.Rp; P.Np = B.Rp; P.ns = A.ns; P.symmetric = symmetric ? 1 : 0;
    P.Ea = A.E; P.Eb = B.E; P.C = C; P.ldc = ldc; P.inner = 0; P.a_row0 = 0; P.accumulate = 1;
    const int ntm = (A.R + BM - 1) / BM, ntn = (B.R + BN - 1) / BN;
    int tiles = 0;
    for (int mt = 0; mt < ntm; mt++) tiles += symmetric ? std::max(0, ntn - (BM / BN) * mt) : ntn;
    if (symmetric && ntn < (BM / BN) * (ntm - 1) + 1) throw std::runtime_error("i8gemm_ar_acc: symmetric product needs a square output");
    const int nkb = A.Kp / BK;
    const int kb_lim = int32_kblocks(A, B);
    if (kb_lim < 1) throw std::runtime_error("i8gemm_ar_acc: slice count too large for exact int32 slice-pair sums");
    if (kb_per > kb_lim) throw std::runtime_error("i8gemm_ar_acc: K range too long for exact int32 slice-pair sums");
    if (kb_per > 0) {
        P.kb_per = std::min(kb_per, nkb);
    } else {
        // K ranges: >= 8 K blocks each; among those the count that wastes the least of the last wave of the persistent grid
        const int ks_min = (nkb + kb_lim - 1) / kb_lim;
        int best = ks_min; double best_eff = -1.0;
        for (int ks = ks_min; ks <= std::max(ks_min, nkb / 8); ks++) {
            const int per = (nkb + ks - 1) / ks, kse = (nkb + per - 1) / per;
            const long items = (long)tiles * kse;
            const double eff = (double)items / ((double)nsm * ((items + nsm - 1) / nsm));
            if (eff > best_eff + 1e-9) { best_eff = eff; best = kse; }
            if (items > 12L * nsm) break;
        }
        P.kb_per = (nkb + best - 1) / best;
    }
    P.ksplit = (nkb + P.kb_per - 1) / P.kb_per;
    P.ntiles = tiles;
    const long items = (long)tiles * P.ksplit;
    launch((unsigned)std::min<long>(items, nsm), ta, tb, P, st);
}

}  // namespace i8g
}  // namespace b200jk
#endif

// Self-test of the int8-slice engine on host buffers (include/b200jk.h): slicing kernels, stage-1 and stage-2 GEMM, outputs
// copied back whole (pads included) so that tests can compare them bit for bit with a model of the engine.
extern "C" int b200jk_i8engine_test(b200jk_handle h, b200jk_i8test* t)
{
    if (!h) return 1;
    if (!t) { set_err(h, "b200jk_i8engine_test: no arguments"); return 1; }
#ifndef B200JK_EMULATE
    std::vector<void*> tmp;
    auto alloc = [&](size_t n) { void* p = dev_alloc(n); tmp.push_back(p); return p; };
    b200jk::i8g::SliceStack SA, SB, SY;
    int rc = 0;
    try {
        using namespace b200jk::i8g;
        const int ns = t->ns, k = t->k, ra = t->ra, rb = t->rb;
        if (ns < 1 || ns > MAXS) throw std::runtime_error("ns out of range");
        if (!t->a || ra < 1 || k < 1 || t->stage < 0 || t->stage > 2) throw std::runtime_error("bad operand A or stage");
        if (t->stage > 0 && (!t->b || rb < 1)) throw std::runtime_error("bad operand B");
        CK(cudaSetDevice(h->device));
        cudaStream_t st = h->stream;
        float* d_norm2 = nullptr;
        if (t->packed) {
            const long npair = (long)k * (k + 1) / 2;
            double* dA = (double*)alloc((size_t)ra * npair * 8);
            h2d(dA, t->a, (size_t)ra * npair * 8, st);
            int* d_rowexp = (int*)alloc((size_t)ra * k * 4);
            d_norm2 = (float*)alloc((size_t)ra * k * 4);
            packed_rowexp(dA, npair, k, ra, d_rowexp, d_norm2, st);
            split_packed(SA, dA, npair, k, ra, d_rowexp, ns, st);
            if (t->rowexp) d2h(t->rowexp, d_rowexp, (size_t)ra * k * 4, st);
            if (t->rownorm2) d2h(t->rownorm2, d_norm2, (size_t)ra * k * 4, st);
        } else {
            double* dA = (double*)alloc((size_t)ra * k * 8);
            h2d(dA, t->a, (size_t)ra * k * 8, st);
            if (t->a_rowmax) {     // maxima as a producer would leave them: bit patterns of non-negative doubles
                split_rows_prepare(SA, ra, k, ns, st);
                h2d(SA.maxbits, t->a_rowmax, (size_t)ra * 8, st);
                split_rows_premax(SA, dA, k, ra, k, ns, st);
            } else {
                split_rows(SA, dA, k, ra, k, ns, st);
            }
        }
        if (t->qa) d2h(t->qa, SA.q, (size_t)ns * SA.Rp * SA.Kp, st);
        if (t->ea) d2h(t->ea, SA.E, (size_t)SA.Rp * 4, st);
        double* dB = nullptr;
        if (t->stage > 0) {
            dB = (double*)alloc((size_t)rb * k * 8);
            h2d(dB, t->b, (size_t)rb * k * 8, st);
            split_rows(SB, dB, k, rb, k, ns, st);
            if (t->qb) d2h(t->qb, SB.q, (size_t)ns * SB.Rp * SB.Kp, st);
            if (t->eb) d2h(t->eb, SB.E, (size_t)SB.Rp * 4, st);
        }
        const int rows = t->stage == 1 ? (t->inner > 0 ? t->inner : t->m) : ra;
        if (t->stage == 1 && t->y_ncolp > 0) {
            if (!t->packed || t->inner != k || t->a_row0 % k || t->m % k || t->m < k)
                throw std::runtime_error("fused Y slices need a packed A and whole blocks of tensor rows");
            double* d_cmax2 = (double*)alloc(8);
            colnorm_max(dB, k, rb, k, d_cmax2, st);
            y_prepare(SY, k, t->m / k, t->y_ncolp, ns, d_norm2 + t->a_row0, d_cmax2, st);
            gemm_ar(SA, t->a_row0, t->m, SB, nullptr, 0, t->inner, st, nullptr, &SY, t->y_ncolp);
            if (t->qy) d2h(t->qy, SY.q, (size_t)ns * SY.Rp * SY.Kp, st);
            if (t->ey) d2h(t->ey, SY.E, (size_t)SY.Rp * 4, st);
        } else if (t->stage > 0) {
            if (t->stage == 1 && (t->m < 1 || t->inner < 0)) throw std::runtime_error("bad row block");
            const long ldc = (t->stage == 1 && t->inner > 0) ? (long)((t->m + t->inner - 1) / t->inner) * rb : rb;
            double* dC = (double*)alloc((size_t)rows * ldc * 8);
            dev_zero(dC, (size_t)rows * ldc * 8, st);
            unsigned long long* d_rm = nullptr;
            if (t->stage == 1 && t->rowmax) { d_rm = (unsigned long long*)alloc((size_t)rows * 8); dev_zero(d_rm, (size_t)rows * 8, st); }
            if (t->stage == 1) gemm_ar(SA, t->a_row0, t->m, SB, dC, ldc, t->inner, st, d_rm);
            else gemm_ar_acc(SA, SB, dC, rb, t->symmetric != 0, st, t->kb_per);
            if (t->c) d2h(t->c, dC, (size_t)rows * ldc * 8, st);
            if (d_rm) d2h(t->rowmax, d_rm, (size_t)rows * 8, st);
        }
        CK(cudaStreamSynchronize(st));
    } catch (std::exception& e) { set_err(h, e.what()); rc = 2; }
    SA.release(); SB.release(); SY.release();
    for (void* p : tmp) dev_free(p);
    return rc;
#else
    set_err(h, "the tensor-core GEMM is not emulated on the CPU");
    return 3;
#endif
}

// C = A B^T through the int8-slice tensor-core path; A [M,K], B [N,K], C [M,N] host fp64 (self-test / tests).
// symmetric: only the upper triangle of C (M == N) is computed, the rest stays zero.
extern "C" int b200jk_i8gemm_test(b200jk_handle h, int M, int N, int K, const double* A, const double* B, double* C, int ns,
                                  int symmetric)
{
    b200jk_i8test t{};
    t.stage = 2; t.ns = ns; t.a = A; t.ra = M; t.k = K; t.b = B; t.rb = N; t.symmetric = symmetric; t.c = C;
    return b200jk_i8engine_test(h, &t);
}
