// i8gemm_host.hpp — host interface of the int8-slice tensor-core GEMM (i8gemm.cu)
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
namespace b200jk {
namespace i8g {
struct SliceStack {      // [ns][Rp][Kp] int8 slices + per-row exponents, device resident
    int8_t* q = nullptr; int* E = nullptr;
    int R = 0, K = 0, Rp = 0, Kp = 0, ns = 0;
    size_t cap = 0; int ecap = 0;
    unsigned long long* maxbits = nullptr; size_t maxbits_cap = 0;
    long zeroed_for = 0;      // shape key for which the pads were last zeroed (y_prepare)
    int dmax = 64;            // largest |digit|: 64 for balanced digits, 127 for the mantissa digits of split_packed (ns <= 7)
    void alloc(int rows, int k, int ns);
    void release();
};
void split_rows(SliceStack& S, const double* X, long ldx, int rows, int k, int ns, cudaStream_t st);
void split_rows_into(SliceStack& S, int row0, const double* X, long ldx, int rows, cudaStream_t st);
// the DF tensor straight from its packed rows cderi[P][a(a+1)/2+b] (no fp64 unpacked copy): per-row exponents of the unpacked
// rows (P, a), then their int8 slices
// Packed DF rows of length npair; with col_of (pair-screened rows, i8gemm.cuh (3)) element t of the packed triangle is column
// col_of[t] of the row, or 0 when col_of[t] < 0.
void packed_rowexp(const double* cderi, long npair, int nao, int nr, int* rowexp, float* rownorm2, cudaStream_t st,
                   const int* col_of = nullptr);
void colnorm_max(const double* X, long ldx, int nrows, int k, double* cmax2, cudaStream_t st);
void y_prepare(SliceStack& S, int nao, int nr, int ncolp, int ns, const float* rownorm2_block, const double* cmax2, cudaStream_t st);
void split_packed_into(SliceStack& S, int out_row0, const double* cderi, long npair, int nao, int nr, const int* rowexp, cudaStream_t st,
                       const int* col_of = nullptr);
void split_packed(SliceStack& S, const double* cderi, long npair, int nao, int nr, const int* rowexp, int ns, cudaStream_t st,
                  const int* col_of = nullptr);
// Yout != nullptr: stage 1 writes the int8 slices of Y (columns (P, i), i padded to y_ncolp) instead of fp64 C
void gemm_ar(const SliceStack& A, int a_row0, int M, const SliceStack& B, double* C, long ldc, int inner, cudaStream_t st,
             unsigned long long* rowmax = nullptr, const SliceStack* Yout = nullptr, int y_ncolp = 0);
void split_rows_prepare(SliceStack& S, int rows, int k, int ns, cudaStream_t st);
void split_rows_premax(SliceStack& S, const double* X, long ldx, int rows, int k, int ns, cudaStream_t st);
// C[m*ldc + n] += A B^T (stage 2 of DF-K); upper triangle only when symmetric.  kb_per > 0 forces K ranges of kb_per K blocks
// (tests); 0 chooses them to fill whole waves, never longer than the int32 bound allows
void gemm_ar_acc(const SliceStack& A, const SliceStack& B, double* C, long ldc, bool symmetric, cudaStream_t st, int kb_per = 0);
}  // namespace i8g
}  // namespace b200jk
