// b200jk.cu — host side of libb200jk.so (C ABI in include/b200jk.h): 4-center direct J/K path.
// With -DB200JK_EMULATE the same file builds with g++ into a CPU SIMT emulation used ONLY by
// tests/ to exercise the host logic and kernel arithmetic without a GPU; the product library is
// always the nvcc build and never falls back to the CPU.
#include "host_common.hpp"
#include "jk_classes.cuh"

namespace {

void ensure_workspace(b200jk_handle h, int n_dm)
{
    if ((size_t)n_dm <= h->ws_ndm) return;
    for (double** p : {&h->d_dm_sph, &h->d_out_sph, &h->d_dmj, &h->d_dmk, &h->d_vj, &h->d_vk}) { dev_free(*p); *p = nullptr; }
    size_t ns2 = (size_t)h->nsph * h->nsph, nc2 = (size_t)h->ncart * h->ncart;
    h->d_dm_sph = (double*)dev_alloc(ns2 * n_dm * 8);
    h->d_out_sph = (double*)dev_alloc(ns2 * n_dm * 8 * 2);
    h->d_dmj = (double*)dev_alloc(nc2 * n_dm * 8);
    h->d_dmk = (double*)dev_alloc(nc2 * n_dm * 8 * 2);
    h->d_vj = (double*)dev_alloc(nc2 * n_dm * 8);
    h->d_vk = (double*)dev_alloc(nc2 * n_dm * 8 * 2);
    h->ws_ndm = n_dm;
}

}  // namespace

// ------------------------------------------------------------------------------------------------
extern "C" const char* b200jk_version(void)
{
#ifdef B200JK_EMULATE
    return "b200jk 0.1 (CPU SIMT emulation — tests only)";
#else
    return "b200jk 0.1 (sm_90a)";
#endif
}

extern "C" const char* b200jk_last_error(b200jk_handle h) { return h ? h->err.c_str() : "null handle"; }

extern "C" int b200jk_create(b200jk_handle* out, const int32_t* atm, int natm, const int32_t* bas, int nbas,
                             const double* env, int nenv, int device)
{
    return b200jk_create2(out, atm, natm, bas, nbas, env, nenv, device, 0);
}

extern "C" int b200jk_create2(b200jk_handle* out, const int32_t* atm, int natm, const int32_t* bas, int nbas,
                              const double* env, int nenv, int device, int cart)
{
    if (!out) return 1;
    *out = nullptr;
    b200jk_handle h = new b200jk_handle_s();
    try {
        h->device = device;
        h->cart = cart ? 1 : 0;
#ifndef B200JK_EMULATE
        int ndev = 0;
        if (cudaGetDeviceCount(&ndev) != cudaSuccess || ndev == 0)
            throw std::runtime_error("no CUDA device: libb200jk has no CPU fallback");
        CK(cudaSetDevice(device));
        CK(cudaStreamCreate(&h->own_stream));
        h->stream = h->own_stream;
        CK(cudaEventCreate(&h->ev0));
        CK(cudaEventCreate(&h->ev1));
        CK(cudaEventCreateWithFlags(&h->ev_in, cudaEventDisableTiming));
        h->side.resize(8); h->side_ev.resize(8);
        {
            // B200JK_LAUNCH_ORDER=1 (tuning experiment): the second half of the side streams gets the highest priority; the cheap,
            // latency-bound classes are launched there FIRST so that they run under the big classes instead of alone at the end
            int lo = 0, hi = 0;
            CK(cudaDeviceGetStreamPriorityRange(&lo, &hi));
            const bool pri = getenv("B200JK_LAUNCH_ORDER") && atoi(getenv("B200JK_LAUNCH_ORDER")) == 1;
            for (size_t i = 0; i < h->side.size(); i++)
                CK(cudaStreamCreateWithPriority(&h->side[i], cudaStreamNonBlocking, (pri && i >= h->side.size() / 2) ? hi : lo));
        }
        for (auto& e : h->side_ev) CK(cudaEventCreateWithFlags(&e, cudaEventDisableTiming));
#endif
        (void)natm; (void)nenv;
        // ---- device shells: general contractions are split into segmented shells
        std::vector<DevShell> tmp;
        int sph = 0;
        for (int ib = 0; ib < nbas; ib++) {
            const int32_t* b = bas + ib * BAS_SLOTS;
            int l = b[ANG_OF], np = b[NPRIM_OF], nc = b[NCTR_OF];
            if (l > LAO_MAX) throw std::runtime_error("angular momentum > f is not supported on the 4-center path");
            const double* r = env + atm[b[ATOM_OF] * ATM_SLOTS + PTR_COORD];
            for (int c = 0; c < nc; c++) {
                DevShell s;
                const int nf = h->cart ? ncart(l) : 2 * l + 1;
                s.l = l; s.ref_shell = ib; s.sph_off = sph + c * nf; s.cart_off = 0;
                s.r[0] = r[0]; s.r[1] = r[1]; s.r[2] = r[2];
                for (int p = 0; p < np; p++) {
                    double cf = env[b[PTR_COEFF] + c * np + p];
                    if (cf != 0.0) { s.e.push_back(env[b[PTR_EXP] + p]); s.c.push_back(cf); }
                }
                s.nprim = (int)s.e.size();
                tmp.push_back(s);
            }
            sph += nc * (h->cart ? ncart(l) : 2 * l + 1);
        }
        h->nsph = sph;
        h->nbas_ref = nbas;
        std::stable_sort(tmp.begin(), tmp.end(), [](const DevShell& a, const DevShell& b) { return a.l < b.l; });
        int co = 0;
        for (auto& s : tmp) { s.cart_off = co; co += ncart(s.l); }
        h->ncart = co;
        h->sh = tmp;
        h->nsh = (int)tmp.size();

        // ---- AO transform tables
        std::vector<int> cart_sh(h->ncart), cart_comp(h->ncart), sph_sh(h->nsph), sph_m(h->nsph), sh_l(h->nsh), sh_cart(h->nsh),
            sh_sph(h->nsh);
        for (int i = 0; i < h->nsh; i++) {
            const DevShell& s = h->sh[i];
            sh_l[i] = s.l; sh_cart[i] = s.cart_off; sh_sph[i] = s.sph_off;
            for (int a = 0; a < ncart(s.l); a++) { cart_sh[s.cart_off + a] = i; cart_comp[s.cart_off + a] = a; }
            for (int m = 0; m < (h->cart ? ncart(s.l) : 2 * s.l + 1); m++) { sph_sh[s.sph_off + m] = i; sph_m[s.sph_off + m] = m; }
            h->ref_shell_of.push_back(s.ref_shell);
        }
        std::vector<double> c2s;
        std::vector<int> c2s_off;
        for (int l = 0; l <= LMAX; l++) {
            c2s_off.push_back((int)c2s.size());
            auto T = h->cart ? make_c2c(l) : make_c2s(l);
            c2s.insert(c2s.end(), T.begin(), T.end());
        }
        h->d_cart_sh = upload(cart_sh); h->d_cart_comp = upload(cart_comp);
        h->d_sph_sh = upload(sph_sh); h->d_sph_m = upload(sph_m);
        h->d_sh_l = upload(sh_l); h->d_sh_cart = upload(sh_cart); h->d_sh_sph = upload(sh_sph);
        h->d_c2s = upload(c2s); h->d_c2s_off = upload(c2s_off);
        for (int l = 0; l <= LMAX; l++) h->c2s_off[l] = c2s_off[l];

        // ---- Rys tables
        {
            const double* blob = (const double*)b200jk_rys_blob;
            size_t nd = b200jk_rys_blob_size / 8;
            if ((int)blob[0] != RYS_NMAX || (int)blob[1] != RYS_DEG || (int)blob[2] != RYS_NINT)
                throw std::runtime_error("rys table header mismatch");
            // device layout: [hermite (NMAX(NMAX+1) doubles)] [pad] [chebyshev rows, 32-byte aligned for 256-bit loads]
            const size_t nherm = RYS_NMAX * (RYS_NMAX + 1), ncheb = nd - 5 - nherm;
            const size_t cheb_off = (nherm + 3) / 4 * 4;
            h->d_rys = (double*)dev_alloc((cheb_off + ncheb) * 8);
            h2d(h->d_rys, blob + 5, nherm * 8);
            h2d(h->d_rys + cheb_off, blob + 5 + nherm, ncheb * 8);
            h->tb.herm = h->d_rys;
            h->tb.cheb = h->d_rys + cheb_off;
        }

        const double expcutoff = (nenv > 0) ? env[0] : 0.0;
        // ---- shell pairs and primitive pairs per class
        for (int la = 0; la <= LAO_MAX; la++)
            for (int lb = 0; lb <= la; lb++) { h->pc[pair_class_id(la, lb)].la = la; h->pc[pair_class_id(la, lb)].lb = lb; }
        for (int i = 0; i < h->nsh; i++)
            for (int j = 0; j <= i; j++) {
                const DevShell &a = h->sh[i], &b = h->sh[j];  // sorted by l => a.l >= b.l
                PairClass& P = h->pc[pair_class_id(a.l, b.l)];
                ShellPair sp{};
                sp.ABx = a.r[0] - b.r[0]; sp.ABy = a.r[1] - b.r[1]; sp.ABz = a.r[2] - b.r[2];
                double r2 = sp.ABx * sp.ABx + sp.ABy * sp.ABy + sp.ABz * sp.ABz;
                sp.ish = i; sp.jsh = j; sp.i0 = a.cart_off; sp.j0 = b.cart_off; sp.same = (i == j);
                sp.prim_off = (int)h->prims.size();
                int np = 0;
                for (int pa = 0; pa < a.nprim; pa++)
                    for (int pb = 0; pb < b.nprim; pb++) {
                        double ea = a.e[pa], eb = b.e[pb], p = ea + eb;
                        double cc = a.c[pa] * b.c[pb] * std::exp(-ea * eb / p * r2);
                        if (std::fabs(cc) < PRIM_CUT) continue;
                        // env[PTR_EXPCUTOFF] (slot 0, pyscf/gto/mole.py:58-88, :3065-3078): the caller's cutoff on the Gaussian-product
                        // exponent of a primitive pair; 0 = library default (here: the coefficient-aware PRIM_CUT above)
                        if (expcutoff > 0.0 && ea * eb / p * r2 > expcutoff) continue;
                        PrimPair pp;
                        pp.p = p;
                        pp.Px = (ea * a.r[0] + eb * b.r[0]) / p; pp.Py = (ea * a.r[1] + eb * b.r[1]) / p; pp.Pz = (ea * a.r[2] + eb * b.r[2]) / p;
                        pp.PAx = pp.Px - a.r[0]; pp.PAy = pp.Py - a.r[1]; pp.PAz = pp.Pz - a.r[2];
                        pp.cc = cc / p * 5.914967172795612486;  // sqrt(2 pi^(5/2)) folded in, see phase_roots
                        h->prims.push_back(pp);
                        np++;
                    }
                sp.nprim = np;
                sp.q = 0.0;
                if (np > 0) P.all.push_back(sp);
            }
        h->d_prims = upload(h->prims);
        int npairs = 0;
        for (int c = 0; c < NPC; c++) { h->pc[c].d_all = upload(h->pc[c].all); npairs += (int)h->pc[c].all.size(); }
        h->d_dmc = (double*)dev_alloc((size_t)h->nsh * h->nsh * 8);
        h->d_counters = (unsigned long long*)dev_alloc(16);
        h->stats.n_dev_shells = h->nsh; h->stats.n_cart = h->ncart; h->stats.n_sph = h->nsph; h->stats.n_pairs = npairs;
        dev_sync();
    } catch (std::exception& e) {
        // keep the handle so the caller can read the message
        h->err = e.what();
        *out = h;
        return 2;
    }
    *out = h;
    return 0;
}

extern "C" int b200jk_destroy(b200jk_handle h)
{
    if (!h) return 0;
    dev_free(h->d_prims); dev_free(h->d_rys);
    for (int c = 0; c < NPC; c++) { dev_free(h->pc[c].d_all); dev_free(h->pc[c].d_kept); }
    dev_free(h->d_cart_sh); dev_free(h->d_cart_comp); dev_free(h->d_sph_sh); dev_free(h->d_sph_m);
    dev_free(h->d_sh_l); dev_free(h->d_sh_cart); dev_free(h->d_sh_sph); dev_free(h->d_c2s); dev_free(h->d_c2s_off);
    dev_free(h->d_dm_sph); dev_free(h->d_out_sph); dev_free(h->d_dmj); dev_free(h->d_dmk); dev_free(h->d_vj); dev_free(h->d_vk);
    dev_free(h->d_dmc); dev_free(h->d_counters); dev_free(h->d_eri);
    if (h->df && h->df_free) h->df_free(h->df);
#ifndef B200JK_EMULATE
    if (h->ev0) cudaEventDestroy(h->ev0);
    if (h->ev1) cudaEventDestroy(h->ev1);
    if (h->own_stream) cudaStreamDestroy(h->own_stream);
    for (auto& s : h->side) cudaStreamDestroy(s);
    for (auto& e : h->side_ev) cudaEventDestroy(e);
    for (auto& e : h->cls_ev) cudaEventDestroy(e);
    if (h->ev_in) cudaEventDestroy(h->ev_in);
#endif
    delete h;
    return 0;
}

extern "C" int b200jk_set_screening(b200jk_handle h, double tol, double omega)
{
    if (!h) return 1;
    try {
        h->tol = tol; h->omega = omega;
        double qmax = 0.0;
        for (int c = 0; c < NPC; c++) {
            PairClass& P = h->pc[c];
            if (P.all.empty()) continue;
            // the reference's bound: normalised real-spherical functions (exact for every l, optimizer.c:408-454)
            const long ne = (long)ncart(P.la) * ncart(P.lb);
            const long chunk = std::max<long>(1, (256L << 20) / (ne * ne * 8));     // <= 256 MB of scratch per launch
            double* scratch = (double*)dev_alloc((size_t)std::min<long>(chunk, (long)P.all.size()) * ne * ne * 8);
            for (long i0 = 0; i0 < (long)P.all.size(); i0 += chunk) {
                long n = std::min<long>(chunk, (long)P.all.size() - i0);
                SchwarzSphFn fn{P.d_all + i0, h->d_prims, h->tb, omega, P.la, P.lb, h->d_c2s + h->c2s_off[P.la], h->d_c2s + h->c2s_off[P.lb], scratch,
                                h->cart ? ncart(P.la) : 2 * P.la + 1, h->cart ? ncart(P.lb) : 2 * P.lb + 1};
                launch_1d(n, fn);
                dev_sync();
            }
            dev_free(scratch);
        }
        dev_sync();
        for (int c = 0; c < NPC; c++) {
            PairClass& P = h->pc[c];
            if (P.all.empty()) continue;
            d2h(P.all.data(), P.d_all, P.all.size() * sizeof(ShellPair));
        }
        dev_sync();
        for (int c = 0; c < NPC; c++)
            for (auto& sp : h->pc[c].all) qmax = std::max(qmax, sp.q);
        for (int c = 0; c < NPC; c++) {
            PairClass& P = h->pc[c];
            P.kept.clear();
            // a pair can only survive q_ij*q_kl > tol if q_ij*qmax > tol (density factors <= O(1) are
            // applied per quartet on device; keep the Schwarz-only bound here, like q_cond in the reference)
            // Deeply contracted pairs are split into sub-pairs of <= MAX_PRIM_PER_PAIR primitive pairs (same shells, same
            // AO block, consecutive primitive ranges).  Integrals are linear in the primitive sum and the unique-quartet
            // rule works on list positions, so (a+b|a+b)/2 = (a|a)/2 + (b|a) + (b|b)/2 is reproduced exactly; it bounds
            // the serial primitive loop of one thread/group (4096 -> 256 for the C 1s x C 1s pairs).
            for (auto& sp : P.all) {
                if (!(sp.q * qmax > tol * 1e-2)) continue;
                for (int p0 = 0; p0 < sp.nprim; p0 += MAX_PRIM_PER_PAIR) {
                    ShellPair sub = sp;
                    sub.prim_off = sp.prim_off + p0;
                    sub.nprim = std::min(MAX_PRIM_PER_PAIR, sp.nprim - p0);
                    P.kept.push_back(sub);
                }
            }
            // batches of kets are homogeneous in primitive count (groups iterate to the longest slot), then by bound
            std::stable_sort(P.kept.begin(), P.kept.end(), [](const ShellPair& a, const ShellPair& b) {
                return a.nprim != b.nprim ? a.nprim > b.nprim : a.q > b.q; });
            dev_free(P.d_kept);
            P.d_kept = upload(P.kept);
        }
        dev_sync();
        h->screened = true;
    } catch (std::exception& e) { set_err(h, e.what()); return 2; }
    return 0;
}

extern "C" int b200jk_get_q_cond(b200jk_handle h, double* q, int nbas)
{
    if (!h || !h->screened) { set_err(h, "call b200jk_set_screening first"); return 1; }
    if (nbas != h->nbas_ref) { set_err(h, "nbas mismatch"); return 1; }
    for (long i = 0; i < (long)nbas * nbas; i++) q[i] = 1e-100;
    for (int c = 0; c < NPC; c++)
        for (auto& sp : h->pc[c].all) {
            int I = h->ref_shell_of[sp.ish], J = h->ref_shell_of[sp.jsh];
            // device bounds are already in the reference's normalisation (spherical, SchwarzSphFn); a general-contracted
            // reference shell takes the maximum over its segments, as CVHFnr_int2e_q_cond does over its nctr blocks
            double v = std::max(sp.q, 1e-100);
            q[(long)I * nbas + J] = std::max(q[(long)I * nbas + J], v);
            q[(long)J * nbas + I] = std::max(q[(long)J * nbas + I], v);
        }
    return 0;
}

static int direct_jk_impl(b200jk_handle h, const double* dm, int n_dm, int nao, int hermi, double* vj, double* vk,
                          bool on_device)
{
    if (!h) return 1;
    try {
        if (!h->screened) throw std::runtime_error("call b200jk_set_screening before b200jk_direct_jk");
        if (nao != h->nsph) throw std::runtime_error("nao does not match the basis of this handle");
        if (n_dm < 1) throw std::runtime_error("n_dm < 1");
        if (!vj && !vk) return 0;
        auto t0 = std::chrono::steady_clock::now();
        ensure_workspace(h, n_dm);
        size_t ns2 = (size_t)h->nsph * h->nsph, nc2 = (size_t)h->ncart * h->ncart;
#ifndef B200JK_EMULATE
        CK(cudaSetDevice(h->device));
        stream_t st = h->stream;
#else
        stream_t st = 0;
#endif
        const double* dsph = dm;
        if (!on_device) { h2d(h->d_dm_sph, dm, ns2 * n_dm * 8, st); dsph = h->d_dm_sph; }
        uint64_t launches = 0;
        // ---- densities in the Cartesian device basis: J sees the symmetric part; K sees sym (and antisym if hermi != 1)
        Sph2CartFn s2c{dsph, h->d_dmj, h->nsph, h->ncart, 0, h->d_cart_sh, h->d_cart_comp, h->d_sh_l, h->d_sh_sph, h->d_c2s_off, h->d_c2s, h->cart};
        int n_dm_k = n_dm;
        const double* dmk = h->d_dmj;
        bool need_sym = (hermi != 2), need_anti = (hermi != 1);
        if (vj || (vk && need_sym)) { launch_1d((long)nc2 * n_dm, s2c, st); launches++; }
        if (vk && need_anti) {
            Sph2CartFn a2c = s2c; a2c.mode = 1;
            if (need_sym) { a2c.dcart = h->d_dmk + nc2 * n_dm; }
            else { a2c.dcart = h->d_dmk; }
            launch_1d((long)nc2 * n_dm, a2c, st); launches++;
            if (need_sym) {
                // [sym ; anti] contiguous in d_dmk
#ifndef B200JK_EMULATE
                CK(cudaMemcpyAsync(h->d_dmk, h->d_dmj, nc2 * n_dm * 8, cudaMemcpyDeviceToDevice, st));
#else
                memcpy(h->d_dmk, h->d_dmj, nc2 * n_dm * 8);
#endif
                n_dm_k = 2 * n_dm;
            }
            dmk = h->d_dmk;
        }
        // dm_cond on the spherical input, the reference's definition (the Schwarz bounds are spherical too)
        DmCondSphFn dc{dsph, n_dm, h->d_dmc, h->nsh, h->nsph, h->d_sh_l, h->d_sh_sph, h->cart};
        launch_1d((long)h->nsh * h->nsh, dc, st); launches++;
        if (vj) dev_zero(h->d_vj, nc2 * n_dm * 8, st);
        if (vk) dev_zero(h->d_vk, nc2 * n_dm_k * 8, st);
        dev_zero(h->d_counters, 16, st);

        KParams P{};
        P.prims = h->d_prims; P.tb = h->tb; P.omega = h->omega; P.tol = h->tol;
        P.dmc = h->d_dmc; P.nsh = h->nsh;
        P.dmj = h->d_dmj; P.dmk = dmk; P.vj = vj ? h->d_vj : nullptr; P.vk = vk ? h->d_vk : nullptr;
        P.n = h->ncart; P.n_dm_j = n_dm; P.n_dm_k = n_dm_k;
        P.counters = h->d_counters;
        P.shard_rank = h->shard_rank; P.shard_world = h->shard_world;
#ifndef B200JK_EMULATE
        CK(cudaEventRecord(h->ev0, st));
#endif
        // classes sorted by estimated work (largest first) and dealt round-robin onto the side streams
        struct Job { int cb, ck; double cost; };
        std::vector<Job> jobs;
        for (int cb = NPC - 1; cb >= 0; cb--)
            for (int ck = cb; ck >= 0; ck--) {
                PairClass &B = h->pc[cb], &K = h->pc[ck];
                if (B.kept.empty() || K.kept.empty()) continue;
                double nq = (double)B.kept.size() * K.kept.size() * (cb == ck ? 0.5 : 1.0);
                double ncomp = (double)ncart(B.la) * ncart(B.lb) * ncart(K.la) * ncart(K.lb);
                double pb = 0, pk = 0;     // primitive pairs on either side -> primitive quartets of the class
                for (const ShellPair& sp : B.kept) pb += sp.nprim;
                for (const ShellPair& sp : K.kept) pk += sp.nprim;
                double pq = pb * pk * (cb == ck ? 0.5 : 1.0);
                int nr = (B.la + B.lb + K.la + K.lb) / 2 + 1;
                // relative class cost (launch/tail + roots + root sum + digestion), a least-squares fit to measured class times
                // of benzene/cc-pVTZ (mean abs error 20 %); only ratios matter: launch order and the multi-GPU balance
                double cost = 0.0976 + 3.14e-9 * pq * nr + 7.6e-10 * pq * nr * ncomp + 2.38e-9 * nq * ncomp + 1.3e-7 * nq;
                if (h->have_costs && h->class_cost[cb * NPC + ck] > 0.0) cost = h->class_cost[cb * NPC + ck];   // measured on this machine
                jobs.push_back({cb, ck, cost});
            }
        std::sort(jobs.begin(), jobs.end(), [](const Job& a, const Job& b) { return a.cost > b.cost; });
        // Multi-GPU partition (reference analogue: omp schedule(dynamic) over AO-block triples, pyscf/lib/vhf/nr_direct.c:429-466).
        // The big classes are split over the ranks by bra pair (round-robin on the cost-sorted lists).  The small ones would shrink
        // to a few CTAs per rank and cost every rank their launch-and-tail latency, so they are given WHOLE to one rank each,
        // longest-processing-time first on the cost model above; every rank takes the same decisions from the same tables.
        std::vector<int> owner(jobs.size(), -1);   // -1: split over all ranks
        if (h->shard_world > 1) {
            const int W = h->shard_world;
            double total = 0;
            for (const Job& jb : jobs) total += jb.cost;
            double cum = 0;
            size_t first_whole = jobs.size();
            // with MEASURED class times (b200jk_set_class_costs) the balance can be trusted: every class that is small against a
            // rank's share goes whole; on the fitted model (20 % mean error) only the cheapest 45 % of the work does
            const double item_cap = h->have_costs ? total / (1.5 * W) : total / (3.0 * W);
            const double cum_cap = h->have_costs ? total : 0.45 * total;
            for (size_t i = jobs.size(); i-- > 0;) {       // from the cheapest class upwards
                if (jobs[i].cost > item_cap || cum + jobs[i].cost > cum_cap) break;
                cum += jobs[i].cost;
                first_whole = i;
            }
            std::vector<double> load(W, 0.0);
            for (size_t i = first_whole; i < jobs.size(); i++) {
                int r = (int)(std::min_element(load.begin(), load.end()) - load.begin());
                owner[i] = r;
                load[r] += jobs[i].cost;
            }
        }
#ifndef B200JK_EMULATE
        CK(cudaEventRecord(h->ev_in, st));
        for (auto& s : h->side) CK(cudaStreamWaitEvent(s, h->ev_in, 0));
#endif
        // launch order and stream of every job: by default descending cost, round-robin over the side streams
        std::vector<size_t> order(jobs.size());
        std::vector<int> job_stream(jobs.size());
        for (size_t i = 0; i < jobs.size(); i++) { order[i] = i; job_stream[i] = (int)(i % 8); }
        {
            static const int launch_order = getenv("B200JK_LAUNCH_ORDER") ? atoi(getenv("B200JK_LAUNCH_ORDER")) : 0;
            if (launch_order == 1 && jobs.size() > 8) {
                double total = 0, cum = 0;
                for (const Job& jb : jobs) total += jb.cost;
                size_t first_small = jobs.size();
                for (size_t i = jobs.size(); i-- > 0;) { if (cum + jobs[i].cost > 0.25 * total) break; cum += jobs[i].cost; first_small = i; }
                size_t n = 0;
                for (size_t i = first_small; i < jobs.size(); i++) { order[n] = i; job_stream[i] = 4 + (int)((i - first_small) % 4); n++; }   // small ones first, high-priority streams
                for (size_t i = 0; i < first_small; i++) { order[n] = i; job_stream[i] = (int)(i % 4); n++; }
            }
        }
        int jn = 0;
        for (size_t oi = 0; oi < jobs.size(); oi++) {
            const size_t ji = order[oi];
            const Job& jb = jobs[ji];
            int cb = jb.cb, ck = jb.ck;
            if (owner[ji] >= 0) {                       // a class given whole to one rank
                if (owner[ji] != h->shard_rank) {
#ifndef B200JK_EMULATE
                    if (h->profile) {     // keep the per-class timers readable: an empty interval
                        if (h->cls_ev.empty()) { h->cls_ev.resize(2 * NPC * NPC); for (auto& e : h->cls_ev) CK(cudaEventCreate(&e)); }
                        CK(cudaEventRecord(h->cls_ev[2 * (cb * NPC + ck)], st));
                        CK(cudaEventRecord(h->cls_ev[2 * (cb * NPC + ck) + 1], st));
                    }
#endif
                    continue;
                }
                P.shard_rank = 0; P.shard_world = 1;
            } else { P.shard_rank = h->shard_rank; P.shard_world = h->shard_world; }
            PairClass &B = h->pc[cb], &K = h->pc[ck];
            // (measured: the thread-per-quartet kernels are also faster on the split lists — balance beats the extra digestions)
            P.bra_pairs = B.d_kept; P.nbra = (int)B.kept.size();
            P.ket_pairs = K.d_kept; P.nket = (int)K.kept.size();
            P.same_class = (cb == ck);
            P.bra_nprim_max = B.kept[0].nprim;  // lists are sorted by primitive count, largest first
            P.ket_nprim_max = K.kept[0].nprim;
#ifndef B200JK_EMULATE
            cudaStream_t ss = h->profile ? st : h->side[job_stream[ji] % h->side.size()];
            if (h->profile) {
                if (h->cls_ev.empty()) { h->cls_ev.resize(2 * NPC * NPC); for (auto& e : h->cls_ev) CK(cudaEventCreate(&e)); }
                CK(cudaEventRecord(h->cls_ev[2 * (cb * NPC + ck)], ss));
            }
            launch_class(cb, ck, P, ss);
            if (h->profile) CK(cudaEventRecord(h->cls_ev[2 * (cb * NPC + ck) + 1], ss));
#else
            launch_class(cb, ck, P, st);
#endif
            launches++;
            jn++;
        }
#ifndef B200JK_EMULATE
        for (size_t i = 0; i < h->side.size(); i++) {
            CK(cudaEventRecord(h->side_ev[i], h->side[i]));
            CK(cudaStreamWaitEvent(st, h->side_ev[i], 0));
        }
        CK(cudaEventRecord(h->ev1, st));
#endif
        // ---- back to the spherical basis with the final symmetrisation
        Cart2SphFn c2s{nullptr, nullptr, h->nsph, h->ncart, 1.0, 0, h->d_sph_sh, h->d_sph_m, h->d_sh_l, h->d_sh_cart, h->d_c2s_off, h->d_c2s};
        double* oj = on_device ? vj : h->d_out_sph;
        double* ok = on_device ? vk : h->d_out_sph + ns2 * n_dm;
        if (vj) { c2s.xcart = h->d_vj; c2s.osph = oj; c2s.sign = 1.0; c2s.accumulate = 0; launch_1d((long)ns2 * n_dm, c2s, st); launches++; }
        if (vk) {
            c2s.osph = ok;
            if (need_sym) { c2s.xcart = h->d_vk; c2s.sign = 1.0; c2s.accumulate = 0; launch_1d((long)ns2 * n_dm, c2s, st); launches++; }
            if (need_anti) {
                c2s.xcart = h->d_vk + (need_sym ? nc2 * n_dm : 0); c2s.sign = -1.0; c2s.accumulate = need_sym ? 1 : 0;
                launch_1d((long)ns2 * n_dm, c2s, st); launches++;
            }
        }
        if (!on_device) {
            if (vj) d2h(vj, oj, ns2 * n_dm * 8, st);
            if (vk) d2h(vk, ok, ns2 * n_dm * 8, st);
        }
        unsigned long long cnt[2] = {0, 0};
        d2h(cnt, h->d_counters, 16, st);
#ifndef B200JK_EMULATE
        CK(cudaStreamSynchronize(st));
        float ms = 0;
        CK(cudaEventElapsedTime(&ms, h->ev0, h->ev1));
        h->stats.ms_kernels = ms;
        if (h->profile)
            for (int cb = 0; cb < NPC; cb++)
                for (int ck = 0; ck <= cb; ck++) {
                    h->class_ms[cb * NPC + ck] = 0.0;
                    if (h->pc[cb].kept.empty() || h->pc[ck].kept.empty()) continue;
                    float cm = 0;
                    CK(cudaEventElapsedTime(&cm, h->cls_ev[2 * (cb * NPC + ck)], h->cls_ev[2 * (cb * NPC + ck) + 1]));
                    h->class_ms[cb * NPC + ck] = cm;
                }
#endif
        auto t1 = std::chrono::steady_clock::now();
        h->stats.ms_total = std::chrono::duration<double, std::milli>(t1 - t0).count();
        h->stats.quartets_computed = cnt[0];
        h->stats.quartets_screened = cnt[1];
        h->stats.kernel_launches = launches;
    } catch (std::exception& e) { set_err(h, e.what()); return 2; }
    return 0;
}

extern "C" int b200jk_direct_jk(b200jk_handle h, const double* dm, int n_dm, int nao, int hermi, double* vj, double* vk)
{
    return direct_jk_impl(h, dm, n_dm, nao, hermi, vj, vk, false);
}
extern "C" int b200jk_direct_jk_device(b200jk_handle h, const double* dm, int n_dm, int nao, int hermi, double* vj, double* vk)
{
    return direct_jk_impl(h, dm, n_dm, nao, hermi, vj, vk, true);
}

// ---- in-core path: J/K from integrals the caller keeps (mf._eri; RHF.get_jk, pyscf/scf/hf.py:2499-2508 -> dot_eri_dm :902-961
// -> _vhf.incore, pyscf/scf/_vhf.py:283-366 -> CVHFnrs8_incore_drv, pyscf/lib/vhf/nr_incore.c:624) ----
extern "C" int b200jk_incore_set_eri(b200jk_handle h, const double* eri, int64_t neri, int nao)
{
    if (!h) return 1;
    try {
        if (!eri || nao < 1) throw std::runtime_error("bad arguments");
        const long npair = (long)nao * (nao + 1) / 2, n4 = (long)nao * nao * nao * nao;
        int sym = 0;
        if (neri == npair * (npair + 1) / 2) sym = 8;
        else if (neri == npair * npair) sym = 4;
        else if (neri == n4) sym = 1;
        if (nao == 1) sym = 1;
        if (!sym) throw std::runtime_error("eri size matches none of s8 / s4 / s1 for this nao (pyscf/scf/hf.py:934-961)");
#ifndef B200JK_EMULATE
        CK(cudaSetDevice(h->device));
#endif
        dev_free(h->d_eri);
        h->d_eri = (double*)dev_alloc((size_t)neri * 8);
        h2d(h->d_eri, eri, (size_t)neri * 8);
        dev_sync();
        h->neri = neri; h->eri_sym = sym;
    } catch (std::exception& e) { set_err(h, e.what()); return 2; }
    return 0;
}

extern "C" int b200jk_incore_jk(b200jk_handle h, const double* dm, int n_dm, int nao, double* vj, double* vk)
{
    if (!h) return 1;
    try {
        if (!h->d_eri) throw std::runtime_error("call b200jk_incore_set_eri before b200jk_incore_jk");
        if (!dm || n_dm < 1 || nao < 1) throw std::runtime_error("bad arguments");
        const long npair = (long)nao * (nao + 1) / 2, n2 = (long)nao * nao;
        const long expect = h->eri_sym == 8 ? npair * (npair + 1) / 2 : (h->eri_sym == 4 ? npair * npair : n2 * n2);
        if (expect != h->neri) throw std::runtime_error("nao does not match the stored integrals");
        if (!vj && !vk) return 0;
#ifndef B200JK_EMULATE
        CK(cudaSetDevice(h->device));
#endif
        stream_t st = 0;
        double* d_dm = (double*)dev_alloc((size_t)n_dm * n2 * 8);
        double* d_j = vj ? (double*)dev_alloc((size_t)n_dm * n2 * 8) : nullptr;
        double* d_k = vk ? (double*)dev_alloc((size_t)n_dm * n2 * 8) : nullptr;
        h2d(d_dm, dm, (size_t)n_dm * n2 * 8, st);
        if (d_j) dev_zero(d_j, (size_t)n_dm * n2 * 8, st);
        if (d_k) dev_zero(d_k, (size_t)n_dm * n2 * 8, st);
        IncoreJKFn fn{h->d_eri, h->eri_sym, nao, npair, d_dm, n_dm, d_j, d_k};
        launch_1d(h->neri, fn, st);
        if (vj) d2h(vj, d_j, (size_t)n_dm * n2 * 8, st);
        if (vk) d2h(vk, d_k, (size_t)n_dm * n2 * 8, st);
        dev_sync();
        dev_free(d_dm); dev_free(d_j); dev_free(d_k);
        h->stats.kernel_launches = 1;
    } catch (std::exception& e) { set_err(h, e.what()); return 2; }
    return 0;
}

extern "C" int b200jk_set_profile(b200jk_handle h, int on) { if (!h) return 1; h->profile = on; return 0; }
extern "C" int b200jk_get_class_times(b200jk_handle h, double* ms, int n)
{
    if (!h || !ms || n != NPC * NPC) return 1;
    memcpy(ms, h->class_ms, sizeof(double) * n);
    return 0;
}

extern "C" int b200jk_class_launch_info(b200jk_handle h, int cb, int ck, int* info, int n)
{
    if (!h) return 1;
    try {
        if (!info || n < B2_LAUNCH_INFO_N || cb < 0 || cb >= NPC || ck < 0 || ck > cb) throw std::runtime_error("bad arguments");
#ifndef B200JK_EMULATE
        CK(cudaSetDevice(h->device));
#endif
        class_info(cb, ck, info);
    } catch (std::exception& e) { set_err(h, e.what()); return 2; }
    return 0;
}

// Measured per-class times (what b200jk_get_class_times returns after a profiled, unsharded build) as the cost table of the
// multi-GPU partition.  Every rank must be given the SAME table (the host layer broadcasts rank 0's: pyscf_b200/parallel.py), since
// the ranks derive the partition independently.  ms == NULL returns to the built-in model.
extern "C" int b200jk_set_class_costs(b200jk_handle h, const double* ms, int n)
{
    if (!h) return 1;
    if (!ms) { h->have_costs = false; return 0; }
    if (n != NPC * NPC) { set_err(h, "class cost table must have 100 entries"); return 1; }
    memcpy(h->class_cost, ms, sizeof(double) * n);
    h->have_costs = true;
    return 0;
}

extern "C" int b200jk_set_shard(b200jk_handle h, int rank, int world)
{
    if (!h || world < 1 || rank < 0 || rank >= world) { set_err(h, "bad shard"); return 1; }
    h->shard_rank = rank; h->shard_world = world;
    return 0;
}

extern "C" int b200jk_set_stream(b200jk_handle h, void* stream)
{
    if (!h) return 1;
#ifndef B200JK_EMULATE
    h->stream = stream ? (cudaStream_t)stream : h->own_stream;
#else
    (void)stream;
#endif
    return 0;
}

#ifndef B200JK_EMULATE
// register-resident DFMA chains: the FP64 roofline denominator of the 4-center path
__global__ void __launch_bounds__(256) fp64_peak_kernel(double* out, int iters)
{
    double a0 = threadIdx.x * 1e-9, a1 = a0 + 1, a2 = a0 + 2, a3 = a0 + 3, a4 = a0 + 4, a5 = a0 + 5, a6 = a0 + 6, a7 = a0 + 7;
    const double m = 1.0000001, c = 1e-7;
    for (int i = 0; i < iters; i++) {
        a0 = fma(a0, m, c); a1 = fma(a1, m, c); a2 = fma(a2, m, c); a3 = fma(a3, m, c);
        a4 = fma(a4, m, c); a5 = fma(a5, m, c); a6 = fma(a6, m, c); a7 = fma(a7, m, c);
    }
    out[blockIdx.x * blockDim.x + threadIdx.x] = a0 + a1 + a2 + a3 + a4 + a5 + a6 + a7;
}
#endif

extern "C" int b200jk_fp64_peak(b200jk_handle h, double* tflops)
{
    if (!h || !tflops) return 1;
#ifndef B200JK_EMULATE
    try {
        CK(cudaSetDevice(h->device));
        int nsm = 0;
        CK(cudaDeviceGetAttribute(&nsm, cudaDevAttrMultiProcessorCount, h->device));
        int blocks = nsm * 8, iters = 1 << 15;
        double* buf = (double*)dev_alloc((size_t)blocks * 256 * 8);
        double best = 0;
        for (int rep = 0; rep < 5; rep++) {
            CK(cudaEventRecord(h->ev0, h->stream));
            fp64_peak_kernel<<<blocks, 256, 0, h->stream>>>(buf, iters);
            CK(cudaEventRecord(h->ev1, h->stream));
            CK(cudaStreamSynchronize(h->stream));
            float ms = 0;
            CK(cudaEventElapsedTime(&ms, h->ev0, h->ev1));
            double tf = 2.0 * 8 * iters * (double)blocks * 256 / (ms * 1e-3) / 1e12;
            if (tf > best) best = tf;
        }
        dev_free(buf);
        *tflops = best;
    } catch (std::exception& e) { set_err(h, e.what()); return 2; }
    return 0;
#else
    *tflops = 0.0;
    return 0;
#endif
}

namespace {
// one x per thread: all n roots and weights, through the same rys_root the integral kernels call
struct RysTestFn {
    RysTables tb; int n; const double* x; double* u; double* w;
    B2_HD void operator()(long i) const
    {
        for (int r = 0; r < n; r++) rys_root(tb, n, r, x[i], u[i * n + r], w[i * n + r]);
    }
};
}  // namespace

extern "C" int b200jk_rys_test(b200jk_handle h, int n, int count, const double* x, double* u, double* w)
{
    if (!h) return 1;
    std::vector<void*> tmp;
    int rc = 0;
    try {
        if (n < 1 || n > RYS_NMAX) throw std::runtime_error("b200jk_rys_test: n out of range 1..9");
        if (count < 0 || (count > 0 && (!x || !u || !w))) throw std::runtime_error("b200jk_rys_test: bad arguments");
        for (int i = 0; i < count; i++)
            if (!(x[i] >= 0.0)) throw std::runtime_error("b200jk_rys_test: x must be >= 0 and not NaN");
        if (count == 0) return 0;
#ifndef B200JK_EMULATE
        CK(cudaSetDevice(h->device));
        stream_t st = h->stream;
#else
        stream_t st = 0;
#endif
        auto alloc = [&](size_t b) { void* p = dev_alloc(b); tmp.push_back(p); return p; };
        double* dx = (double*)alloc((size_t)count * 8);
        double* du = (double*)alloc((size_t)count * n * 8);
        double* dw = (double*)alloc((size_t)count * n * 8);
        h2d(dx, x, (size_t)count * 8, st);
        launch_1d(count, RysTestFn{h->tb, n, dx, du, dw}, st);
        d2h(u, du, (size_t)count * n * 8, st);
        d2h(w, dw, (size_t)count * n * 8, st);
#ifndef B200JK_EMULATE
        CK(cudaStreamSynchronize(st));
#endif
    } catch (std::exception& e) { set_err(h, e.what()); rc = 2; }
    for (void* p : tmp) dev_free(p);
    return rc;
}

extern "C" int b200jk_get_dm_cond_test(b200jk_handle h, double* dmc, int32_t* ao_off, int nsh)
{
    if (!h) return 1;
    try {
        if (!dmc || nsh != h->nsh) throw std::runtime_error("b200jk_get_dm_cond_test: nsh must be the number of device shells");
        if (!h->ws_ndm) throw std::runtime_error("b200jk_get_dm_cond_test: no b200jk_direct_jk call yet");
#ifndef B200JK_EMULATE
        CK(cudaSetDevice(h->device));
#endif
        d2h(dmc, h->d_dmc, (size_t)nsh * nsh * 8);
        dev_sync();
        if (ao_off)
            for (int i = 0; i < nsh; i++) ao_off[i] = h->sh[i].sph_off;
    } catch (std::exception& e) { set_err(h, e.what()); return 2; }
    return 0;
}

extern "C" int b200jk_get_stats(b200jk_handle h, b200jk_stats* out)
{
    if (!h || !out) return 1;
    *out = h->stats;
    return 0;
}

// ---- density fitting entry points live in df.cu; stubs until that translation unit is linked
#ifndef B200JK_HAVE_DF
extern "C" int b200jk_df_build(b200jk_handle h, const int32_t*, int, const int32_t*, int, const double*, int, double, double)
{ set_err(h, "density-fitting path not built into this library"); return 3; }
extern "C" int b200jk_df_jk(b200jk_handle h, const double*, int, int, const double*, int, int, double*, double*)
{ set_err(h, "density-fitting path not built into this library"); return 3; }
extern "C" int b200jk_df_naux(b200jk_handle h, int*)
{ set_err(h, "density-fitting path not built into this library"); return 3; }
#endif
