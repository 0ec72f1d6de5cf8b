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
using ao2mo::BM; using ao2mo::BN; using ao2mo::BK; using ao2mo::NT; using ao2mo::LDC; using ao2mo::PER_T;

constexpr int RT = 256;     // threads of the diagonal sums

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
AO_D double chi_at(const double* chi, long K, long k0, int t) { const long k = k0 + t % BK; return k < K ? chi[k] : 0.0; }
AO_D void scale(double* ra, double cx) { for (int q = 0; q < PER_T; q++) ra[q] *= cx; }

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

// thread t of the diagonal sums: its strided share of log L_PP (the factor's diagonal in M) and of Pi_PP
AO_D void diag_share(const double* M, const double* dg, long N, int t, double* red)
{
    double a = 0.0, b = 0.0;
    for (long P = t; P < N; P += RT) { a += log(M[P * N + P]); b += dg[P]; }
    red[t] = a; red[RT + t] = b;
}
AO_D void red_step(double* red, int t, int s) { if (t < s) { red[t] += red[t + s]; red[RT + t] += red[RT + t + s]; } }

#ifndef B200JK_EMULATE
__global__ void __launch_bounds__(NT) rpa_pi_kernel(Job jb)
{
    __shared__ __align__(128) double sm[ao2mo::SMEM];
    const long m0 = (long)jb.tiles[2 * blockIdx.x] * BM, n0 = (long)jb.tiles[2 * blockIdx.x + 1] * BN;
    const PiGemm& g = jb.g;
    const int t = threadIdx.x, w = t >> 5;
    ao2mo::fr::C c[4][4];
#pragma unroll
    for (int a = 0; a < 4; a++)
#pragma unroll
        for (int b = 0; b < 4; b++) ao2mo::fr::zero(c[a][b]);
    double ra[PER_T], rb[PER_T];
    ao2mo::fetch(g, m0, n0, 0, t, ra, rb);
    double cx = chi_at(jb.chi, g.K, 0, t);
    for (long k0 = 0; k0 < g.K; k0 += BK) {
        scale(ra, cx);
        ao2mo::put<PiGemm>(sm, t, ra, rb);
        __syncthreads();
        if (k0 + BK < g.K) {     // next k step in flight during the MMAs
            ao2mo::fetch(g, m0, n0, k0 + BK, t, ra, rb);
            cx = chi_at(jb.chi, g.K, k0 + BK, t);
        }
        ao2mo::warp_mma(sm, w, c);
        __syncthreads();
    }
    ao2mo::warp_store(sm, w, c);
    __syncthreads();
    pi_epilogue(jb, sm, m0, n0, t);
}

__global__ void __launch_bounds__(RT) rpa_diag_kernel(const double* M, const double* dg, long N, double* out)
{
    __shared__ double red[2 * RT];
    const int t = threadIdx.x;
    diag_share(M, dg, N, t, red);
    __syncthreads();
    for (int s = RT / 2; s > 0; s >>= 1) {
        red_step(red, t, s);
        __syncthreads();
    }
    if (t == 0) { out[0] = 2.0 * red[0]; out[1] = red[RT]; }
}

static void pi_launch(const Job& jb, int ntile, cudaStream_t s)
{
    rpa_pi_kernel<<<ntile, NT, 0, s>>>(jb);
    CK(cudaGetLastError());
}
static void diag_launch(const double* M, const double* dg, long N, double* out, cudaStream_t s)
{
    rpa_diag_kernel<<<1, RT, 0, s>>>(M, dg, N, out);
    CK(cudaGetLastError());
}
#else
// the same CTA code, thread by thread and warp by warp, on the host model of the fragments
static void pi_launch(const Job& jb, int ntile, stream_t)
{
    const PiGemm& g = jb.g;
    std::vector<double> sm(ao2mo::SMEM), ra(NT * PER_T), rb(NT * PER_T), cx(NT);
    std::vector<ao2mo::fr::C> cw(4 * 16);
    typedef ao2mo::fr::C Acc[4][4];
    Acc* c = reinterpret_cast<Acc*>(cw.data());
    for (int x = 0; x < ntile; x++) {
        const long m0 = (long)jb.tiles[2 * x] * BM, n0 = (long)jb.tiles[2 * x + 1] * BN;
        for (ao2mo::fr::C& v : cw) ao2mo::fr::zero(v);
        for (int t = 0; t < NT; t++) {
            ao2mo::fetch(g, m0, n0, 0, t, &ra[t * PER_T], &rb[t * PER_T]);
            cx[t] = chi_at(jb.chi, g.K, 0, t);
        }
        for (long k0 = 0; k0 < g.K; k0 += BK) {
            for (int t = 0; t < NT; t++) {
                scale(&ra[t * PER_T], cx[t]);
                ao2mo::put<PiGemm>(sm.data(), t, &ra[t * PER_T], &rb[t * PER_T]);
            }
            if (k0 + BK < g.K)
                for (int t = 0; t < NT; t++) {
                    ao2mo::fetch(g, m0, n0, k0 + BK, t, &ra[t * PER_T], &rb[t * PER_T]);
                    cx[t] = chi_at(jb.chi, g.K, k0 + BK, t);
                }
            for (int w = 0; w < 4; w++) ao2mo::warp_mma(sm.data(), w, c[w]);
        }
        for (int w = 0; w < 4; w++) ao2mo::warp_store(sm.data(), w, c[w]);
        for (int t = 0; t < NT; t++) pi_epilogue(jb, sm.data(), m0, n0, t);
    }
}
static void diag_launch(const double* M, const double* dg, long N, double* out, stream_t)
{
    std::vector<double> red(2 * RT);
    for (int t = 0; t < RT; t++) diag_share(M, dg, N, t, red.data());
    for (int s = RT / 2; s > 0; s >>= 1)
        for (int t = 0; t < RT; t++) red_step(red.data(), t, s);
    out[0] = 2.0 * red[0]; out[1] = red[RT];
}
#endif

}  // namespace rpak

extern "C" int b200jk_df_rpa(b200jk_handle h, int nspin, const double* const* c_occ, const int* nocc, const double* const* c_vir,
                             const int* nvir, const double* const* e_ov, const double* const* f_ov, int nw, const double* omega,
                             double* logdet, double* trace, double* diel)
{
    if (!h) return 1;
    try {
        DFState* d = h->df;
        if (!d || !d->d_cderi) throw std::runtime_error("call b200jk_df_build (or b200jk_df_set_cderi) before b200jk_df_rpa");
        if (d->build_world != 1)
            throw std::runtime_error("b200jk_df_rpa: a sharded tensor is not supported (Pi needs every auxiliary row of L)");
        if ((nspin != 1 && nspin != 2) || !c_occ || !nocc || !c_vir || !nvir || !e_ov || !f_ov || nw < 1 || !omega || !logdet ||
            !trace || (diel && nw != 1))
            throw std::runtime_error("bad arguments");
        bool active[2] = {false, false};
        for (int s = 0; s < nspin; s++) {
            if (nocc[s] < 0 || nvir[s] < 0) throw std::runtime_error("bad arguments: negative orbital count");
            active[s] = nocc[s] > 0 && nvir[s] > 0;
            if (active[s] && (!c_occ[s] || !c_vir[s] || !e_ov[s] || !f_ov[s])) throw std::runtime_error("bad arguments");
        }
        auto t_start = std::chrono::steady_clock::now();
        const int nao = h->nsph, nrow = d->nrow;
        const long N = nrow;
#ifndef B200JK_EMULATE
        CK(cudaSetDevice(h->device));
        cudaStream_t st = h->stream;
#else
        stream_t st = 0;
#endif
        // stage-1 pairs (co, cv) of the active spins, in spin order: the K segments of Pi
        HalfPair pr[2];
        int npr = 0, na_max = 1;
        long K = 0;
        for (int s = 0; s < nspin; s++)
            if (active[s]) {
                pr[npr] = HalfPair{{c_occ[s], c_vir[s]}, {nocc[s], nvir[s]}, 0, (long)nocc[s] * nvir[s], nullptr, {nullptr, nullptr}};
                na_max = std::max(na_max, std::min(nocc[s], nvir[s]));
                K += pr[npr++].nij;
            }
        const int rb = half_block_rows(nrow, nao, na_max);
#ifndef B200JK_EMULATE
        int lwork = 0;
        CKS(cusolverDnSetStream(d->cusolver, st));
        // the buffer query reads only n and lda; the tensor rows stand in for the matrix, which is not allocated yet
        CKS(cusolverDnDpotrf_bufferSize(d->cusolver, CUBLAS_FILL_MODE_LOWER, (int)N, d->d_cderi, (int)N, &lwork));
#else
        const int lwork = 0;
#endif
        double need = (double)rb * nao * na_max + (double)N * N * (diel ? 2 : 1) + lwork + 3.0 * K + N + 2.0 * nw;
        for (int q = 0; q < npr; q++) need += (double)nrow * pr[q].nij;
        ao2mo_check_fit(8.0 * need, "DF-RPA: the half-transformed integrals L[naux, nocc nvir] of each spin, Pi[naux, naux] and "
                                    "the factorisation workspace");

        std::vector<void*> owned;
        auto alloc = [&](size_t bytes) { void* p = dev_alloc(bytes); owned.push_back(p); return p; };
        try {
            double ms1 = 0.0, ms2 = 0.0, ms3 = 0.0;
            if (npr > 0) {
                for (int q = 0; q < npr; q++) {
                    pr[q].L = (double*)alloc((size_t)std::max(nrow, 1) * pr[q].nij * 8);
                    for (int s = 0; s < 2; s++) {
                        pr[q].dc[s] = (double*)alloc((size_t)nao * pr[q].n[s] * 8);
                        h2d(pr[q].dc[s], pr[q].c[s], (size_t)nao * pr[q].n[s] * 8, st);
                    }
                }
                double* d_Y = (double*)dev_alloc((size_t)rb * nao * na_max * 8);
                try { ms1 = half_transform(d, nao, st, pr, npr, d_Y, rb); } catch (...) { dev_sync(); dev_free(d_Y); throw; }
                dev_sync();
                dev_free(d_Y);
            }
            // e_ov, f_ov of the active spins as one K vector, in the order of the segments
            double* d_e = (double*)alloc((size_t)std::max(K, 1L) * 8);
            double* d_f = (double*)alloc((size_t)std::max(K, 1L) * 8);
            double* d_chi = (double*)alloc((size_t)std::max(K, 1L) * 8);
            for (int s = 0, q = 0; s < nspin; s++)
                if (active[s]) {
                    const long k0 = q ? pr[0].nij : 0;
                    h2d(d_e + k0, e_ov[s], (size_t)pr[q].nij * 8, st);
                    h2d(d_f + k0, f_ov[s], (size_t)pr[q].nij * 8, st);
                    q++;
                }
            double* d_M = (double*)alloc((size_t)N * N * 8);
            double* d_dg = (double*)alloc((size_t)N * 8);
            double* d_diel = diel ? (double*)alloc((size_t)N * N * 8) : nullptr;
            double* d_out = (double*)alloc((size_t)2 * nw * 8);
            int* d_info = (int*)alloc((size_t)nw * 4);
            dev_zero(d_info, (size_t)nw * 4, st);
#ifndef B200JK_EMULATE
            double* d_work = (double*)alloc((size_t)std::max(lwork, 1) * 8);
#endif
            const long nt = (N + ao2mo::BM - 1) / ao2mo::BM;
            std::vector<int> tl;
            for (int A = 0; A < nt; A++)
                for (int B = A; B < nt; B++) { tl.push_back(A); tl.push_back(B); }
            const int ntile = (int)(tl.size() / 2);
            int* d_tiles = (int*)alloc(tl.size() * 4);
            h2d(d_tiles, tl.data(), tl.size() * 4, st);
            const long k1 = npr > 0 ? pr[0].nij : 0, ld1 = npr > 1 ? pr[1].nij : 0;
            const double* L0 = npr > 0 ? pr[0].L : nullptr;
            const double* L1 = npr > 1 ? pr[1].L : nullptr;
            const rpak::Seg seg{L0, L1, k1, ld1};
            rpak::Job jb{rpak::PiGemm{N, N, K, {seg}, {seg}, {}, 0, 0, 0}, d_chi, d_tiles, d_M, d_dg, d_diel};
#ifndef B200JK_EMULATE
            std::vector<cudaEvent_t> ev(3 * (size_t)nw, nullptr);
            for (cudaEvent_t& e : ev) CK(cudaEventCreate(&e));
            try {
                for (int w = 0; w < nw; w++) {
                    CK(cudaEventRecord(ev[3 * w], st));
                    launch_1d(K, rpak::ChiFn{d_e, d_f, omega[w] * omega[w], d_chi}, st);
                    rpak::pi_launch(jb, ntile, st);
                    CK(cudaEventRecord(ev[3 * w + 1], st));
                    CKS(cusolverDnDpotrf(d->cusolver, CUBLAS_FILL_MODE_LOWER, (int)N, d_M, (int)N, d_work, lwork, d_info + w));
                    rpak::diag_launch(d_M, d_dg, N, d_out + 2 * w, st);
                    CK(cudaEventRecord(ev[3 * w + 2], st));
                }
                CK(cudaStreamSynchronize(st));
                for (int w = 0; w < nw; w++) {
                    float t = 0;
                    CK(cudaEventElapsedTime(&t, ev[3 * w], ev[3 * w + 1]));
                    ms2 += t;
                    CK(cudaEventElapsedTime(&t, ev[3 * w + 1], ev[3 * w + 2]));
                    ms3 += t;
                }
            } catch (...) {
                for (cudaEvent_t e : ev) cudaEventDestroy(e);
                throw;
            }
            for (cudaEvent_t e : ev) cudaEventDestroy(e);
#else
            std::vector<double> a((size_t)N * N);
            for (int w = 0; w < nw; w++) {
                launch_1d(K, rpak::ChiFn{d_e, d_f, omega[w] * omega[w], d_chi}, st);
                rpak::pi_launch(jb, ntile, st);
                // cpu_cholesky_lower reads the row-major lower triangle: mirror the upper one that the epilogue wrote
                for (long m = 0; m < N; m++)
                    for (long n = 0; n < N; n++) a[m * N + n] = d_M[std::min(m, n) * N + std::max(m, n)];
                bool ok = true;
                cpu_cholesky_lower(a, (int)N, ok);
                if (!ok) { d_info[w] = 1; continue; }
                for (long P = 0; P < N; P++) d_M[P * N + P] = a[P * N + P];
                rpak::diag_launch(d_M, d_dg, N, d_out + 2 * w, st);
            }
#endif
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
            d->rpa_ms[0] = ms1; d->rpa_ms[1] = ms2; d->rpa_ms[2] = ms3;
        } catch (...) {
            dev_sync();
            for (void* p : owned) dev_free(p);
            throw;
        }
        dev_sync();
        for (void* p : owned) dev_free(p);
        d->rpa_ms[3] = std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now() - t_start).count();
    } catch (std::exception& e) { set_err(h, e.what()); return 2; }
    return 0;
}

extern "C" int b200jk_df_rpa_times(b200jk_handle h, double* ms, int n)
{
    if (!h || !h->df || !ms) { set_err(h, "call b200jk_df_build first"); return 1; }
    for (int i = 0; i < n; i++) ms[i] = i < 4 ? h->df->rpa_ms[i] : 0.0;
    return 0;
}
