// df_mp2.cuh — DF-MP2 energies and amplitudes from the resident tensor (included by df.cu after df_ao2mo.cuh).
//
//   b200jk_df_mp2   DFRMP2 / DFUMP2 kernel   pyscf/mp/dfmp2.py:39-121, dfump2.py:38-166
//                                            (MP2_contract_d, MP2_OS_contract_d, pyscf/lib/mp/mp2.c:89-275)
//
// Stage 1, per spin: L[P, i nvir + a] = C_occ[:, i]^T B_P C_vir[:, a] for every local row P, the s1 pair (co, cv) of ao2mo's
// stage 1 (half_transform), resident on the device.
// Stage 2: one CTA per occupied pair (i, j) and virtual tile pair (A, B) of 64 x 64.  Same spin: i >= j, A <= B; the CTA
// accumulates V[A, B] = L_i[:, A]^T L_j[:, B] and, when A != B, V[B, A] = L_i[:, B]^T L_j[:, A] over K = naux on the ao2mo GEMM
// core: two 64 x 64 DMMA accumulators, each held by its own group of four warps (256 threads; one set of accumulators and
// prefetch registers per thread, as in ao2mo's GEMM, which already needs ~240 registers).  On a diagonal tile pair (A = B) the
// two groups take alternate k steps of V[A, A] and their halves are added in shared memory.  The epilogue stages both tiles in
// shared memory, so each thread holds V_ab and V_ba of its elements and sums, over (a, b) in A x B and, when A != B, in B x A,
//     ed += V_ab t_ab,   ex -= V_ba t_ab,   t_ab = V_ab / (e_i + e_j - e_a - e_b)
// with the pair factor of _MP2_gen_jobs (mp2.c:44-69): 2 for i != j, 1 for i == j.  Opposite spin (UMP2 alpha-beta): every
// (i, j), every tile pair, V[A, B] only, no exchange, one group of warps.  V and (ia|jb) never reach global memory.  With amplitudes the epilogue
// writes t_ab (UMP2 same spin: t_ab - t_ba) for a band of pairs to a device buffer, which band_pipeline copies to the caller.
// Reduction: each CTA sums its threads' (ed, ex) in a fixed tree and stores the result at its own (pair, tile pair) slot of a
// partial array that covers all pairs; one CTA then sums that array in a fixed order.  The energies therefore do not depend on
// the band size, on where the tensor rows live or on the launch order: two calls give the same bits.

namespace mp2k {
using ao2mo::BM; using ao2mo::BN; using ao2mo::BK; using ao2mo::NT; using ao2mo::LDC; using ao2mo::RT;
using ao2mo::SM_AB; using ao2mo::SM_C;

constexpr int SMEM = 2 * SM_C;      // two staged C tiles; the operand tiles of both products (2 SM_AB) sit below them
static_assert(2 * SM_AB <= SMEM, "operands of both products fit in the C staging");

struct NoSt {};
typedef ao2mo::Gemm<ao2mo::TransA, ao2mo::RowsB, NoSt> PairGemm;   // a(m, k) = L_i[k, m], b(k, n) = L_j[k, n]

struct Job {
    const double *La, *Lb; long lda, ldb;     // L of the spin of i and of j: [naux][nocc nvir]
    int nva, nvb, naux;
    const double *eoa, *eob, *eva, *evb;      // orbital energies (device)
    const int* pairs;                         // [npair][2]: (i, j)
    const int* tiles;                         // [ntp][2]: (A, B)
    int ntp, os, t2mode;                      // os: opposite spin; t2mode 1: t_ab, 2: t_ab - t_ba
    double* t2; long p0;                      // amplitudes of pairs [p0, ...): pair p at t2 + (p - p0) nva nvb; nullptr: none
    double* part;                             // [npair][ntp][2]: (ed, -ex) of each CTA
};

AO_D PairGemm pair_gemm(const Job& jb, int i, int j)
{
    return PairGemm{jb.nva, jb.nvb, jb.naux, {jb.La + (long)i * jb.nva, jb.lda}, {jb.Lb + (long)j * jb.nvb, jb.ldb}, {}, 0, 0, 0};
}

// thread t (of T) of the elements (x, y) = (R0 + r, C0 + c) of the staged tile X[r][c] = V_xy; Y[c][r] = V_yx (exchange)
AO_D void epi_tile(const Job& jb, const double* X, const double* Y, long R0, long C0, double eij, int t, int T, double* t2p,
                   double& ed, double& ex)
{
    for (int e = t; e < BM * BN; e += T) {
        const int r = e / BN, c = e % BN;
        const long x = R0 + r, y = C0 + c;
        if (x >= jb.nva || y >= jb.nvb) continue;
        const double v = X[r * LDC + c];
        const double dd = eij - (jb.eva[x] + jb.evb[y]);
        const double tv = v / dd;
        ed += v * tv;
        double tw = tv;
        if (!jb.os) {
            const double w = Y[c * LDC + r];
            ex += w * tv;
            if (jb.t2mode == 2) tw = tv - w / dd;
        }
        if (t2p) t2p[x * jb.nvb + y] = tw;
    }
}

// CTA (pair p, tile pair tp) of T threads after its products: the epilogue of thread t; the tiles are staged at sm (V[A, B])
// and, when two, at sm + SM_C (V[B, A])
AO_D void cta_epilogue(const Job& jb, const double* sm, long p, int i, int j, long A0, long B0, bool two, int t, int T, double* red)
{
    const double eij = jb.eoa[i] + jb.eob[j];
    double* t2p = jb.t2 ? jb.t2 + (p - jb.p0) * (long)jb.nva * jb.nvb : nullptr;
    double ed = 0.0, ex = 0.0;
    epi_tile(jb, sm, two ? sm + SM_C : sm, A0, B0, eij, t, T, t2p, ed, ex);
    if (two) epi_tile(jb, sm + SM_C, sm, B0, A0, eij, t, T, t2p, ed, ex);
    red[t] = ed; red[T + t] = ex;
}
AO_D void cta_store(const Job& jb, const double* red, long p, int tp, int i, int j, int T)
{
    const double fac = (!jb.os && i != j) ? 2.0 : 1.0;
    jb.part[(p * jb.ntp + tp) * 2] = fac * red[0];
    jb.part[(p * jb.ntp + tp) * 2 + 1] = -(fac * red[T]);
}
// threads of a CTA: one group of four warps per accumulator
AO_D constexpr int cta_threads(int os) { return os ? NT : 2 * NT; }
// k steps of group grp: a diagonal same-spin tile pair (split) gives the two groups alternate steps (grp, grp + 2, ...) of its
// one product, else each group takes them all; both groups run the same number of steps (the last one of group 1 may be past K)
AO_D void k_plan(bool split, int grp, long K, long& k_first, long& k_step, long& k_end)
{
    const long nk = (K + BK - 1) / BK;
    k_first = split ? grp * BK : 0;
    k_step = split ? 2 * BK : BK;
    k_end = k_first + (split ? (nk + 1) / 2 : nk) * k_step;
}
// thread t (of T) of the sum of the two staged halves of a split product into the first tile
AO_D void add_halves(double* sm, int t, int T) { for (int e = t; e < BM * LDC; e += T) sm[e] += sm[SM_C + e]; }
// thread t of the final sum: its strided share of n partial (ed, ex)
struct PartShare {
    const double* part; long n;
    AO_D void operator()(int t, double& a, double& b) const { for (long q = t; q < n; q += RT) { a += part[2 * q]; b += part[2 * q + 1]; } }
};

#ifndef B200JK_EMULATE
// group 0 (threads [0, NT)) accumulates V[A, B], group 1 V[B, A]; on a diagonal tile pair they split the k steps of V[A, A]
template <int OS>
__global__ void __launch_bounds__(cta_threads(OS)) mp2_pair_kernel(Job jb, long p_base)
{
    constexpr int T = cta_threads(OS);
    extern __shared__ __align__(128) double sm[];
    __shared__ double red[2 * T];
    const long p = p_base + blockIdx.y;
    const int tp = blockIdx.x;
    const int i = jb.pairs[2 * p], j = jb.pairs[2 * p + 1];
    const long A0 = (long)jb.tiles[2 * tp] * BM, B0 = (long)jb.tiles[2 * tp + 1] * BN;
    const bool two = !OS && A0 != B0, split = !OS && A0 == B0;
    const int t = threadIdx.x, grp = t / NT, tg = t % NT;
    const PairGemm g = pair_gemm(jb, i, j);
    ao2mo::fr::C c[4][4];
    ao2mo::NoHook hk;
    long kf, ks, ke;
    k_plan(split, grp, g.K, kf, ks, ke);
    ao2mo::k_loop(g, grp ? B0 : A0, grp ? A0 : B0, kf, ks, ke, sm + grp * SM_AB, tg, hk, c);
    ao2mo::warp_store(sm + grp * SM_C, tg >> 5, c);
    __syncthreads();
    if (split) {
        add_halves(sm, t, T);
        __syncthreads();
    }
    cta_epilogue(jb, sm, p, i, j, A0, B0, two, t, T, red);
    __syncthreads();
    for (int s = T / 2; s > 0; s >>= 1) {
        ao2mo::red_step(red, t, s, T);
        __syncthreads();
    }
    if (t == 0) cta_store(jb, red, p, tp, i, j, T);
}

// pairs [p0, p1) of the job, every tile pair
static void pair_launch(const Job& jb, long p0, long p1, cudaStream_t s)
{
    if (p1 <= p0 || jb.ntp <= 0) return;
    const int bytes = SMEM * 8;
    if (jb.os) CK(cudaFuncSetAttribute(mp2_pair_kernel<1>, cudaFuncAttributeMaxDynamicSharedMemorySize, bytes));
    else CK(cudaFuncSetAttribute(mp2_pair_kernel<0>, cudaFuncAttributeMaxDynamicSharedMemorySize, bytes));
    for (long y0 = p0; y0 < p1; y0 += 65535) {
        const dim3 grid((unsigned)jb.ntp, (unsigned)std::min<long>(65535, p1 - y0));
        if (jb.os) mp2_pair_kernel<1><<<grid, cta_threads(1), bytes, s>>>(jb, y0);
        else mp2_pair_kernel<0><<<grid, cta_threads(0), bytes, s>>>(jb, y0);
    }
    CK(cudaGetLastError());
}
#else
// the same CTA code on the host model; the two groups of warps run one after the other (their operand tiles and accumulators
// are disjoint until the stores)
static void pair_launch(const Job& jb, long p0, long p1, stream_t)
{
    const int T = cta_threads(jb.os);
    std::vector<double> sm(SMEM), red(2 * T);
    ao2mo::Acc c[8];     // c[grp * 4 + w]
    for (long p = p0; p < p1; p++)
        for (int tp = 0; tp < jb.ntp; tp++) {
            const int i = jb.pairs[2 * p], j = jb.pairs[2 * p + 1];
            const long A0 = (long)jb.tiles[2 * tp] * BM, B0 = (long)jb.tiles[2 * tp + 1] * BN;
            const bool two = !jb.os && A0 != B0, split = !jb.os && A0 == B0;
            const PairGemm g = pair_gemm(jb, i, j);
            for (int grp = 0; grp < T / NT; grp++) {
                long kf, ks, ke;
                k_plan(split, grp, g.K, kf, ks, ke);
                ao2mo::k_loop(g, grp ? B0 : A0, grp ? A0 : B0, kf, ks, ke, sm.data() + grp * SM_AB, ao2mo::NoHook{}, c + 4 * grp);
            }
            for (int grp = 0; grp < T / NT; grp++)
                for (int w = 0; w < 4; w++) ao2mo::warp_store(sm.data() + grp * SM_C, w, c[grp * 4 + w]);
            if (split)
                for (int t = 0; t < T; t++) add_halves(sm.data(), t, T);
            for (int t = 0; t < T; t++) cta_epilogue(jb, sm.data(), p, i, j, A0, B0, two, t, T, red.data());
            for (int s = T / 2; s > 0; s >>= 1)
                for (int t = 0; t < T; t++) ao2mo::red_step(red.data(), t, s, T);
            cta_store(jb, red.data(), p, tp, i, j, T);
        }
}
#endif

// amplitudes of the pairs [p0, p0 + np) from a band at src into the caller's t2: same spin [no][no][nv][nv] with
// t2[j, i] = t2[i, j]^T (mp2.c:162-167), opposite spin [noa][nob][nva][nvb] in pair order
static void scatter_t2(const int* pairs, long p0, long np, const double* src, double* t2, int no, int nva, int nvb, bool os)
{
    const long nvv = (long)nva * nvb;
    if (os) { ao2mo::par_memcpy(t2 + p0 * nvv, src, (size_t)np * nvv * 8); return; }
    auto one = [&](long q) {
        const int i = pairs[2 * (p0 + q)], j = pairs[2 * (p0 + q) + 1];
        const double* blk = src + q * nvv;
        memcpy(t2 + ((long)i * no + j) * nvv, blk, (size_t)nvv * 8);
        if (i != j) {
            double* tr = t2 + ((long)j * no + i) * nvv;
            for (int a = 0; a < nva; a++)
                for (int b = 0; b < nvb; b++) tr[(long)b * nva + a] = blk[(long)a * nvb + b];
        }
    };
    const int nt = (int)std::min<long>(8, std::max<long>(1, np * nvv / (4L << 20)));
    if (nt == 1) { for (long q = 0; q < np; q++) one(q); return; }
    std::vector<std::thread> th;
    for (int k = 0; k < nt; k++) th.emplace_back([=]() { for (long q = k; q < np; q += nt) one(q); });
    for (std::thread& x : th) x.join();
}

}  // namespace mp2k

extern "C" int b200jk_df_mp2(b200jk_handle h, int nspin, const double* const* c_occ, const int* nocc, const double* const* c_vir,
                             const int* nvir, const double* const* e_occ, const double* const* e_vir, double* e_out,
                             double* const* t2)
{
    if (!h) return 1;
    try {
        MoCall c(h, "b200jk_df_mp2", " (the pair energies are not linear in the local rows)");
        DFState* d = c.d;
        const stream_t st = c.st;
        if ((nspin != 1 && nspin != 2) || !c_occ || !nocc || !c_vir || !nvir || !e_occ || !e_vir || !e_out)
            throw std::runtime_error("bad arguments");
        ActiveSpins sp(nspin, c_occ, nocc, c_vir, nvir, e_occ, e_vir);
        const int nao = h->nsph, nrow = d->nrow;
        // jobs: (spin of i, spin of j, opposite spin, t2 mode, caller's t2 block)
        struct JobSpec { int sa, sb, os, mode; double* t2; long npair, ntp; };
        std::vector<JobSpec> specs;
        if (nspin == 1) specs.push_back({0, 0, 0, 1, t2 ? t2[0] : nullptr, 0, 0});
        else {
            specs.push_back({0, 0, 0, 2, t2 ? t2[0] : nullptr, 0, 0});
            specs.push_back({1, 1, 0, 2, t2 ? t2[2] : nullptr, 0, 0});
            specs.push_back({0, 1, 1, 1, t2 ? t2[1] : nullptr, 0, 0});
        }
        auto ntile = [](int nv) { return (long)(nv + ao2mo::BM - 1) / ao2mo::BM; };
        double need = 0.0, part_total = 0.0, band_max = 0.0;
        for (JobSpec& js : specs) {
            if (!sp.active(js.sa) || !sp.active(js.sb)) continue;
            js.npair = js.os ? (long)nocc[js.sa] * nocc[js.sb] : (long)nocc[js.sa] * (nocc[js.sa] + 1) / 2;
            js.ntp = js.os ? ntile(nvir[js.sa]) * ntile(nvir[js.sb]) : ntile(nvir[js.sa]) * (ntile(nvir[js.sa]) + 1) / 2;
            part_total += 2.0 * js.npair * js.ntp;
            const long nvv = (long)nvir[js.sa] * nvir[js.sb];
            if (js.t2) band_max = std::max(band_max, (double)ao2mo_band_rows(d, js.npair, nvv * 8) * nvv);
        }
        const int rb = half_block_rows(nrow, nao, sp.na_max);
        for (int q = 0; q < sp.npr; q++) need += (double)nrow * sp.pr[q].nij;
        need += std::max((double)rb * nao * sp.na_max, part_total + 2.0 * band_max);
        ao2mo_check_fit(8.0 * need, "DF-MP2: the half-transformed integrals L[naux, nocc nvir] of each spin with their work buffers");

        const double ms1 = half_transform(c, nao, sp.pr, sp.npr, rb, sp.na_max);
        double ms2 = 0.0;
        double* d_eo[2] = {nullptr, nullptr};
        double* d_ev[2] = {nullptr, nullptr};
        for (int s = 0; s < nspin; s++)
            if (sp.active(s)) {
                d_eo[s] = (double*)c.alloc((size_t)nocc[s] * 8);
                d_ev[s] = (double*)c.alloc((size_t)nvir[s] * 8);
                h2d(d_eo[s], e_occ[s], (size_t)nocc[s] * 8, st);
                h2d(d_ev[s], e_vir[s], (size_t)nvir[s] * 8, st);
            }
        double* d_sums = (double*)c.alloc(2 * specs.size() * 8);
        dev_zero(d_sums, 2 * specs.size() * 8, st);
        StageTimer tm;     // the jobs without amplitudes; band_pipeline times the others
        std::vector<std::vector<int>> pair_lists(specs.size());
        for (size_t k = 0; k < specs.size(); k++) {
            const JobSpec& js = specs[k];
            if (js.npair == 0) continue;
            const int sa = js.sa, sb = js.sb, nva = nvir[sa], nvb = nvir[sb];
            const HalfPair &pa = sp.pr[sp.pr_of[sa]], &pb = sp.pr[sp.pr_of[sb]];
            // pairs i-major (consecutive CTAs share L_i), tile pairs in row order
            std::vector<int>& pl = pair_lists[k];
            for (int i = 0; i < nocc[sa]; i++)
                for (int j = 0; j < (js.os ? nocc[sb] : i + 1); j++) { pl.push_back(i); pl.push_back(j); }
            std::vector<int> tl;
            for (int A = 0; A < ntile(nva); A++)
                for (int B = js.os ? 0 : A; B < ntile(nvb); B++) { tl.push_back(A); tl.push_back(B); }
            int* d_pairs = (int*)c.alloc(pl.size() * 4);
            int* d_tiles = (int*)c.alloc(tl.size() * 4);
            h2d(d_pairs, pl.data(), pl.size() * 4, st);
            h2d(d_tiles, tl.data(), tl.size() * 4, st);
            double* d_part = (double*)c.alloc((size_t)js.npair * js.ntp * 2 * 8);
            mp2k::Job jb{pa.L, pb.L, pa.nij, pb.nij, nva, nvb, nrow, d_eo[sa], d_eo[sb], d_ev[sa], d_ev[sb], d_pairs, d_tiles,
                         (int)js.ntp, js.os, js.mode, nullptr, 0, d_part};
            const mp2k::PartShare share{d_part, js.npair * js.ntp};
            if (!js.t2) {
                tm.mark(0, st);
                mp2k::pair_launch(jb, 0, js.npair, st);
                ao2mo::tree_sum(share, d_sums + 2 * k, st);
                tm.mark(-1, st);
            } else {
                const long nvv = (long)nva * nvb, band = ao2mo_band_rows(d, js.npair, nvv * 8);
                const int nbands = (int)((js.npair + band - 1) / band);
                ao2mo::band_pipeline(d, st, nbands, (size_t)band * nvv * 8, [&](int b, double* buf) -> size_t {
                    const long p0 = (long)b * band, p1 = std::min(js.npair, p0 + band);
                    mp2k::Job jt = jb;
                    jt.t2 = buf; jt.p0 = p0;
                    mp2k::pair_launch(jt, p0, p1, st);
                    if (b == nbands - 1) ao2mo::tree_sum(share, d_sums + 2 * k, st);
                    return (size_t)(p1 - p0) * nvv * 8;
                }, [&](int b, const void* src, size_t n) {
                    mp2k::scatter_t2(pl.data(), (long)b * band, (long)(n / 8 / nvv), (const double*)src, js.t2, nocc[sa], nva, nvb,
                                     js.os != 0);
                }, ms2);
            }
        }
        std::vector<double> sums(2 * specs.size());
        d2h(sums.data(), d_sums, sums.size() * 8, st);
        dev_sync();
        double ms_nt = 0.0;
        tm.read(&ms_nt, nullptr, 1);
        // the reference's combination: RMP2 dfmp2.py:109-119, UMP2 dfump2.py:119,154,164 (ex is stored with its sign)
        if (nspin == 1) { e_out[0] = sums[0] + sums[1]; e_out[1] = sums[0]; }
        else {
            double ess = 0.0;
            ess += (sums[0] + sums[1]) * 0.5;
            ess += (sums[2] + sums[3]) * 0.5;
            e_out[0] = ess; e_out[1] = sums[4];
        }
        d->mp2_ms[0] = ms1; d->mp2_ms[1] = ms2 + ms_nt;
        d->mp2_ms[2] = c.finish();
    } catch (std::exception& e) { set_err(h, e.what()); return 2; }
    return 0;
}

extern "C" int b200jk_df_mp2_times(b200jk_handle h, double* ms, int n) { return mo_times(h, &DFState::mp2_ms, ms, n); }
