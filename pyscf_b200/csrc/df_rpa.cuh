// df_rpa.cuh — direct-RPA correlation energy from the resident tensor (included by df.cu after df_mp2.cuh).
//
//   b200jk_df_rpa   RPA / URPA kernel   pyscf/gw/rpa.py:43-130, urpa.py:41-72
//
// Stage 1, per spin s: L_s[P, i nvir_s + a] = C_occ[:, i]^T B_P C_vir[:, a] for every row P (half_transform, the s1 pair
// (co, cv) that DF-MP2 uses), resident on the device.
// Stage 2, one frequency w at a time, into one [naux][naux] buffer M:
//     chi_s[ia] = 2 e_ov f_ov / (w^2 + e_ov^2)                                  (rpa.py:118, urpa.py:62)
//     Pi[P, Q]  = sum_s sum_ia L_s[P, ia] chi_s[ia] L_s[Q, ia]                  (rpa.py:121-127)
// on the ao2mo GEMM core: a(m, k) = chi[k] L[m, k], b(k, n) = L[n, k], the two spins two segments of one K in the same CTA (no
// atomics, no split K: Pi is bit-reproducible).  Only the CTA tiles with n0 >= m0 run; the epilogue writes M[m][n] = delta_mn
// - Pi[m, n] (row-major upper triangle = column-major lower triangle, what potrf LOWER reads), keeps diag(Pi) and, for the
// dielectric matrix itself, writes Pi to both triangles of a second buffer.  Then potrf factors M = L L^T in place and one CTA
// sums logdet = 2 sum_P log L_PP and tr Pi = sum_P Pi_PP in a fixed order.  The caller adds w_n / 2pi (logdet + trace) over the
// frequencies (rpa.py:80-84); log(det(.)) of the reference is replaced by the Cholesky form, which is finite where det overflows.
// The emulation build runs the same CTA code on the host fragment model and factors with cpu_cholesky_lower.

namespace rpak {
using ao2mo::BM; using ao2mo::BN; using ao2mo::BK; using ao2mo::NT; using ao2mo::LDC; using ao2mo::PER_T; using ao2mo::RT;

// L[r, k] over K = [spin 0 | spin 1]: L0 [naux][k1], L1 [naux][ld1]
struct Seg {
    const double *L0, *L1; long k1, ld1;
    B2_HD double at(long r, long k) const { return k < k1 ? L0[r * k1 + k] : L1[r * ld1 + (k - k1)]; }
};
// a(m, k) = L[m, k] (chi[k] is applied when the operand is put to shared memory), b(k, n) = L[n, k]
struct SegA {
    Seg s;
    static constexpr bool MFAST = false;
    B2_HD double operator()(long m, long k) const { return s.at(m, k); }
};
struct SegB {
    Seg s;
    static constexpr bool NFAST = false;
    B2_HD double operator()(long k, long n) const { return s.at(n, k); }
};
struct NoSt {};
typedef ao2mo::Gemm<SegA, SegB, NoSt> PiGemm;
// every A element a thread stages in one k step has k = k0 + t % BK (MFAST = false), so one chi value per thread and k step;
// it is loaded with the operands, one step ahead, and multiplied in at the put, after the MMAs that hide the loads
static_assert(NT % BK == 0, "one k per thread in the A operand");
struct ChiHook {
    const double* chi; long K; double cx;
    AO_D void at(long k0, int t) { const long k = k0 + t % BK; cx = k < K ? chi[k] : 0.0; }
    AO_D void apply(double* ra) const { for (int q = 0; q < PER_T; q++) ra[q] *= cx; }
};

struct Job {
    PiGemm g;           // M = N = naux, K = sum_s nocc_s nvir_s
    const double* chi;  // [K]
    const int* tiles;   // [ntile][2]: (m tile, n tile), n tile >= m tile
    double* M;          // [naux][naux]: I - Pi, upper triangle (row-major)
    double* dg;         // [naux]: Pi_PP
    double* diel;       // nullptr, or [naux][naux]: Pi, both triangles
};

struct ChiFn {
    const double *e, *f; double w2; double* chi;
    B2_HD void operator()(long k) const { chi[k] = 2.0 * e[k] * f[k] / (w2 + e[k] * e[k]); }
};

// thread t of the epilogue of the tile at (m0, n0), staged at sm
AO_D void pi_epilogue(const Job& jb, const double* sm, long m0, long n0, int t)
{
    const long N = jb.g.M;
    for (int e = t; e < BM * BN; e += NT) {
        const int r = e / BN, c = e % BN;
        const long m = m0 + r, n = n0 + c;
        if (m >= N || n >= N) continue;
        const double v = sm[r * LDC + c];
        jb.M[m * N + n] = (m == n ? 1.0 : 0.0) - v;
        if (m == n) jb.dg[m] = v;
        // Pi from the upper triangle only: on a diagonal tile (m, n) and (n, m) differ in the last bits and must not both write
        if (jb.diel && n >= m) { jb.diel[m * N + n] = v; jb.diel[n * N + m] = v; }
    }
}

// thread t of the diagonal sums: its strided share of 2 log L_PP (the factor's diagonal in M) and of Pi_PP
struct DiagShare {
    const double *M, *dg; long N;
    AO_D void operator()(int t, double& a, double& b) const
    {
        for (long P = t; P < N; P += RT) { a += log(M[P * N + P]); b += dg[P]; }
        a *= 2.0;
    }
};

#ifndef B200JK_EMULATE
__global__ void __launch_bounds__(NT) rpa_pi_kernel(Job jb)
{
    __shared__ __align__(128) double sm[ao2mo::SMEM];
    const long m0 = (long)jb.tiles[2 * blockIdx.x] * BM, n0 = (long)jb.tiles[2 * blockIdx.x + 1] * BN;
    const int t = threadIdx.x;
    ao2mo::fr::C c[4][4];
    ChiHook hk{jb.chi, jb.g.K, 0.0};
    ao2mo::k_loop(jb.g, m0, n0, 0, BK, jb.g.K, sm, t, hk, c);
    ao2mo::warp_store(sm, t >> 5, c);
    __syncthreads();
    pi_epilogue(jb, sm, m0, n0, t);
}

static void pi_launch(const Job& jb, int ntile, cudaStream_t s)
{
    rpa_pi_kernel<<<ntile, NT, 0, s>>>(jb);
    CK(cudaGetLastError());
}
#else
// the same CTA code on the host model of the fragments
static void pi_launch(const Job& jb, int ntile, stream_t)
{
    std::vector<double> sm(ao2mo::SMEM);
    ao2mo::Acc c[4];
    for (int x = 0; x < ntile; x++) {
        const long m0 = (long)jb.tiles[2 * x] * BM, n0 = (long)jb.tiles[2 * x + 1] * BN;
        ao2mo::k_loop(jb.g, m0, n0, 0, BK, jb.g.K, sm.data(), ChiHook{jb.chi, jb.g.K, 0.0}, c);
        for (int w = 0; w < 4; w++) ao2mo::warp_store(sm.data(), w, c[w]);
        for (int t = 0; t < NT; t++) pi_epilogue(jb, sm.data(), m0, n0, t);
    }
}
#endif

}  // namespace rpak

extern "C" int b200jk_df_rpa(b200jk_handle h, int nspin, const double* const* c_occ, const int* nocc, const double* const* c_vir,
                             const int* nvir, const double* const* e_ov, const double* const* f_ov, int nw, const double* omega,
                             double* logdet, double* trace, double* diel)
{
    if (!h) return 1;
    try {
        MoCall c(h, "b200jk_df_rpa", " (Pi needs every auxiliary row of L)");
        DFState* d = c.d;
        const stream_t st = c.st;
        if ((nspin != 1 && nspin != 2) || !c_occ || !nocc || !c_vir || !nvir || !e_ov || !f_ov || nw < 1 || !omega || !logdet ||
            !trace || (diel && nw != 1))
            throw std::runtime_error("bad arguments");
        // the active spins in spin order: the K segments of Pi
        ActiveSpins sp(nspin, c_occ, nocc, c_vir, nvir, e_ov, f_ov);
        const int nao = h->nsph, nrow = d->nrow;
        const long N = nrow;
        long K = 0;
        for (int q = 0; q < sp.npr; q++) K += sp.pr[q].nij;
        const int rb = half_block_rows(nrow, nao, sp.na_max);
#ifndef B200JK_EMULATE
        int lwork = 0;
        CKS(cusolverDnSetStream(d->cusolver, st));
        // the buffer query reads only n and lda; the tensor rows stand in for the matrix, which is not allocated yet
        CKS(cusolverDnDpotrf_bufferSize(d->cusolver, CUBLAS_FILL_MODE_LOWER, (int)N, d->d_cderi, (int)N, &lwork));
#else
        const int lwork = 0;
#endif
        double need = (double)rb * nao * sp.na_max + (double)N * N * (diel ? 2 : 1) + lwork + 3.0 * K + N + 2.0 * nw;
        for (int q = 0; q < sp.npr; q++) need += (double)nrow * sp.pr[q].nij;
        ao2mo_check_fit(8.0 * need, "DF-RPA: the half-transformed integrals L[naux, nocc nvir] of each spin, Pi[naux, naux] and "
                                    "the factorisation workspace");

        const double ms1 = half_transform(c, nao, sp.pr, sp.npr, rb, sp.na_max);
        // e_ov, f_ov of the active spins as one K vector, in the order of the segments
        double* d_e = (double*)c.alloc((size_t)std::max(K, 1L) * 8);
        double* d_f = (double*)c.alloc((size_t)std::max(K, 1L) * 8);
        double* d_chi = (double*)c.alloc((size_t)std::max(K, 1L) * 8);
        for (int s = 0; s < nspin; s++)
            if (sp.active(s)) {
                const int q = sp.pr_of[s];
                const long k0 = q ? sp.pr[0].nij : 0;
                h2d(d_e + k0, e_ov[s], (size_t)sp.pr[q].nij * 8, st);
                h2d(d_f + k0, f_ov[s], (size_t)sp.pr[q].nij * 8, st);
            }
        double* d_M = (double*)c.alloc((size_t)N * N * 8);
        double* d_dg = (double*)c.alloc((size_t)N * 8);
        double* d_diel = diel ? (double*)c.alloc((size_t)N * N * 8) : nullptr;
        double* d_out = (double*)c.alloc((size_t)2 * nw * 8);
        int* d_info = (int*)c.alloc((size_t)nw * 4);
        dev_zero(d_info, (size_t)nw * 4, st);
        const long nt = (N + ao2mo::BM - 1) / ao2mo::BM;
        std::vector<int> tl;
        for (int A = 0; A < nt; A++)
            for (int B = A; B < nt; B++) { tl.push_back(A); tl.push_back(B); }
        const int ntile = (int)(tl.size() / 2);
        int* d_tiles = (int*)c.alloc(tl.size() * 4);
        h2d(d_tiles, tl.data(), tl.size() * 4, st);
        const long k1 = sp.npr > 0 ? sp.pr[0].nij : 0, ld1 = sp.npr > 1 ? sp.pr[1].nij : 0;
        const double* L0 = sp.npr > 0 ? sp.pr[0].L : nullptr;
        const double* L1 = sp.npr > 1 ? sp.pr[1].L : nullptr;
        const rpak::Seg seg{L0, L1, k1, ld1};
        rpak::Job jb{rpak::PiGemm{N, N, K, {seg}, {seg}, {}, 0, 0, 0}, d_chi, d_tiles, d_M, d_dg, d_diel};
        // M = L L^T in place (d_info[w] != 0: not positive definite)
#ifndef B200JK_EMULATE
        double* d_work = (double*)c.alloc((size_t)std::max(lwork, 1) * 8);
        auto factor = [&](int w) {
            CKS(cusolverDnDpotrf(d->cusolver, CUBLAS_FILL_MODE_LOWER, (int)N, d_M, (int)N, d_work, lwork, d_info + w));
        };
#else
        std::vector<double> a((size_t)N * N);
        auto factor = [&](int w) {
            // cpu_cholesky_lower reads the row-major lower triangle: mirror the upper one that the epilogue wrote
            for (long m = 0; m < N; m++)
                for (long n = 0; n < N; n++) a[m * N + n] = d_M[std::min(m, n) * N + std::max(m, n)];
            bool ok = true;
            cpu_cholesky_lower(a, (int)N, ok);
            if (!ok) { d_info[w] = 1; return; }
            for (long P = 0; P < N; P++) d_M[P * N + P] = a[P * N + P];
        };
#endif
        StageTimer tm;     // [0] chi and Pi, [1] factorisation and diagonal sums
        for (int w = 0; w < nw; w++) {
            tm.mark(0, st);
            launch_1d(K, rpak::ChiFn{d_e, d_f, omega[w] * omega[w], d_chi}, st);
            rpak::pi_launch(jb, ntile, st);
            tm.mark(1, st);
            factor(w);
            ao2mo::tree_sum(rpak::DiagShare{d_M, d_dg, N}, d_out + 2 * w, st);
            tm.mark(-1, st);
        }
        std::vector<int> info(nw);
        std::vector<double> out((size_t)2 * nw);
        d2h(info.data(), d_info, (size_t)nw * 4, st);
        d2h(out.data(), d_out, out.size() * 8, st);
        if (diel) d2h(diel, d_diel, (size_t)N * N * 8, st);
        dev_sync();
        for (int w = 0; w < nw; w++) {
            if (info[w] == 0) continue;
            char buf[400];
            snprintf(buf, sizeof buf, "DF-RPA: I - Pi(omega) is not positive definite at omega = %.10g (potrf info %d); RPA is not "
                     "well-defined for degenerate systems or for occupied orbitals above virtual ones", omega[w], info[w]);
            throw std::runtime_error(buf);
        }
        for (int w = 0; w < nw; w++) { logdet[w] = out[2 * w]; trace[w] = out[2 * w + 1]; }
        double ms23[2];
        tm.read(ms23, nullptr, 2);
        d->rpa_ms[0] = ms1; d->rpa_ms[1] = ms23[0]; d->rpa_ms[2] = ms23[1];
        d->rpa_ms[3] = c.finish();
    } catch (std::exception& e) { set_err(h, e.what()); return 2; }
    return 0;
}

extern "C" int b200jk_df_rpa_times(b200jk_handle h, double* ms, int n) { return mo_times(h, &DFState::rpa_ms, ms, n); }
