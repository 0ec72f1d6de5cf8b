// df.cu — density-fitting path of libb200jk.so.
//
//   b200jk_df_build : cderi[naux, nao(nao+1)/2] = L^-1 (P|ij)     <- incore.cholesky_eri, pyscf/df/incore.py:129-220
//                     (P|Q), (ij|P) from the Rys kernels in df_block.cuh, Cholesky/TRSM on device
//                     (eigendecomposition fallback with `lindep`, incore.py:150-158,263-270)
//   b200jk_df_jk    : J = cderi^T (cderi . dmtril) ; K = sum_P (P|.i)(P|.i)^T  <- df_jk.get_jk, pyscf/df/df_jk.py:280-413
//   b200jk_df_ao2mo, b200jk_df_get_ao_eri : MO / AO integrals from the tensor      <- DF.ao2mo / get_eri, pyscf/df/df.py:269-296
//                     (df_ao2mo.cuh, FP64 tensor-core GEMMs)
//   b200jk_df_mp2   : DF-MP2 energies and amplitudes from the tensor            <- DFRMP2 / DFUMP2, pyscf/mp/dfmp2.py:39-121,
//                     (df_mp2.cuh, the same GEMM core)                              dfump2.py:38-166
//   b200jk_df_rpa   : direct-RPA correlation energy from the tensor             <- RPA / URPA, pyscf/gw/rpa.py:43-130,
//                     (df_rpa.cuh, the same GEMM core + potrf)                      urpa.py:41-72
// The tensor stays resident in HBM in the reference's own layout (row P, packed lower triangle mu>=nu).
// The four MO consumers of the tensor (ao2mo, get_ao_eri, DF-MP2, DF-RPA) share one call harness (MoCall), one stage 1
// (half_transform) and one CTA k loop on the FP64 GEMM core (ao2mo::k_loop); all of them, get_ao_eri included, visit the host
// rows through RowSplit::walk.
#include "host_common.hpp"
#include "df_classes.cuh"

#include <functional>

#ifndef B200JK_EMULATE
#include <cublas_v2.h>
#include <cusolverDn.h>
#include "i8gemm_host.hpp"
#define CKB(call)                                                                                  \
    do {                                                                                           \
        cublasStatus_t s_ = (call);                                                                \
        if (s_ != CUBLAS_STATUS_SUCCESS) {                                                         \
            char buf_[256];                                                                        \
            snprintf(buf_, sizeof buf_, "%s failed: cublas status %d (%s:%d)", #call, (int)s_, __FILE__, __LINE__); \
            throw std::runtime_error(buf_);                                                        \
        }                                                                                          \
    } while (0)
#define CKS(call)                                                                                  \
    do {                                                                                           \
        cusolverStatus_t s_ = (call);                                                              \
        if (s_ != CUSOLVER_STATUS_SUCCESS) {                                                       \
            char buf_[256];                                                                        \
            snprintf(buf_, sizeof buf_, "%s failed: cusolver status %d (%s:%d)", #call, (int)s_, __FILE__, __LINE__); \
            throw std::runtime_error(buf_);                                                        \
        }                                                                                          \
    } while (0)
#endif

using namespace b200jk;

// ---- device / host row split ---------------------------------------------------------------------
// bytes of int8 slices per packed row, and what the K build needs besides the tensor: the per-block slice stack and 12 GB of
// workspaces (the reserve the slice-residency decision keeps)
static size_t slice_row_bytes(int nao, int ns) { return (size_t)ns * nao * (((size_t)nao + 127) / 128 * 128); }
static size_t k_reserve_bytes(int nao, int kb, int ns) { return (size_t)(kb + 1) * slice_row_bytes(nao, ns) + (12UL << 30); }
// rows per K block of a rank holding nloc rows: the block unpacked to nao x nao takes at most 2 GiB
static int k_block_rows(int nao, int nloc)
{
    return (int)std::max<long>(1, std::min<long>(std::max(nloc, 1), (2048L << 20) / ((long)nao * nao * 8)));
}
// rows [lo, hi) of n that rank `rank` of `world` owns
static void shard_range(long n, int rank, int world, int& lo, int& hi)
{
    lo = (int)(n * rank / world); hi = (int)(n * (rank + 1) / world);
}

// MemAvailable of /proc/meminfo in bytes (0 when it cannot be read)
static size_t host_mem_available()
{
    FILE* f = fopen("/proc/meminfo", "r");
    if (!f) return 0;
    char line[256];
    size_t kb = 0;
    while (fgets(line, sizeof line, f))
        if (sscanf(line, "MemAvailable: %zu kB", &kb) == 1) break;
    fclose(f);
    return kb * 1024;
}

// Where the local rows of the tensor live: rows [0, n_dev) in HBM (DFState::d_cderi), rows [n_dev, nrow) in pinned host memory.
// The host rows are streamed through the two device staging buffers d_stage (stage_rows rows each) once per J/K or MO transform
// call.  n_dev == nrow when the tensor fits next to the K workspaces.
struct RowSplit {
    int n_dev = 0, stage_rows = 0;
    long ld = 0;                       // row length in doubles
    double* h_cderi = nullptr;
    double* d_stage[2] = {nullptr, nullptr};
    int64_t bytes = 0; double copy_ms = 0.0, exposed_ms = 0.0;   // last timed walk (b200jk_df_stream_stats)
    int timed_blocks = 0;
#ifndef B200JK_EMULATE
    // H2D copies run on cp_stream; per staged block, events at copy start / end and around the wait of the compute stream
    // (exposed copy time); ev_free[slot] marks the compute on a staging buffer done
    cudaStream_t cp_stream = nullptr;
    cudaEvent_t ev_start = nullptr, ev_free[2] = {nullptr, nullptr};
    std::vector<cudaEvent_t> blk_ev;
#endif

    ~RowSplit()
    {
#ifndef B200JK_EMULATE
        for (cudaEvent_t e : blk_ev) cudaEventDestroy(e);
        for (cudaEvent_t e : {ev_start, ev_free[0], ev_free[1]}) if (e) cudaEventDestroy(e);
        if (cp_stream) cudaStreamDestroy(cp_stream);
        if (h_cderi) cudaFreeHost(h_cderi);
#else
        free(h_cderi);
#endif
        dev_free(d_stage[0]); dev_free(d_stage[1]);
    }

    // Decide how many of this rank's nloc rows of ld_ doubles stay in HBM and allocate them in *dev (zero-filled on request), the
    // pinned host rows and the two staging buffers.  With the automatic split (h->df_dev_rows = -1) every row stays on the device
    // when the tensor fits next to the K reserve; otherwise the device keeps as many rows as leave room for that reserve and the
    // staging buffers.  The host part is checked against MemAvailable before it is allocated.  Returns an empty string on
    // success, else the error (the caller frees the state).
    std::string plan(b200jk_handle h, int nloc, long ld_, int k_slices, bool zero_fill, double** dev, stream_t st)
    {
        const int nao = h->nsph;
        ld = ld_;
        const size_t rowb = (size_t)ld * 8;
        const size_t stage_cap = std::max<size_t>(1, std::min<size_t>(std::max(nloc, 1), (1UL << 30) / rowb));   // rows in 1 GiB
        long nd = nloc;
        if (h->df_dev_rows >= 0) nd = std::min<long>(nloc, h->df_dev_rows);
#ifndef B200JK_EMULATE
        else {
            size_t freeb = 0, totb = 0;
            CK(cudaMemGetInfo(&freeb, &totb));
            const double reserve = (double)k_reserve_bytes(nao, k_block_rows(nao, nloc), k_slices);
            if ((double)nloc * rowb + reserve > (double)freeb) {
                const double avail = (double)freeb - reserve - 2.0 * stage_cap * rowb - (double)(1UL << 30);
                nd = avail > 0 ? std::min<long>(nloc, (long)(avail / rowb)) : 0;
            }
        }
#endif
        const long n_host = nloc - nd;
        if (n_host > 0) {
            const size_t hbytes = (size_t)n_host * rowb, avail = host_mem_available();
            if (avail && (double)hbytes > 0.9 * (double)avail - (double)(2UL << 30)) {
                char buf[320];
                snprintf(buf, sizeof buf, "the DF tensor does not fit: %ld of its %d rows (%.1f GB) exceed the device and need pinned "
                         "host memory, but MemAvailable is %.1f GB", n_host, nloc, hbytes / 1e9, avail / 1e9);
                return buf;
            }
        }
        n_dev = (int)nd;
        *dev = (double*)dev_alloc((size_t)std::max<long>(nd, 1) * rowb);
        if (zero_fill) dev_zero(*dev, (size_t)std::max<long>(nd, 1) * rowb, st);
        if (n_host > 0) {
            stage_rows = (int)std::min<long>((long)stage_cap, n_host);
#ifndef B200JK_EMULATE
            CK(cudaHostAlloc((void**)&h_cderi, (size_t)n_host * rowb, cudaHostAllocDefault));
#else
            h_cderi = (double*)malloc((size_t)n_host * rowb);
            if (!h_cderi) throw std::runtime_error("host rows of the DF tensor: out of memory");
#endif
            for (double*& s : d_stage) s = (double*)dev_alloc((size_t)stage_rows * rowb);
        }
        return "";
    }

    double* host_row(long r) const { return h_cderi + (size_t)(r - n_dev) * ld; }
    // end of the device rows of the local range [r_lo, r_hi): rows [r_lo, dev_end) are in HBM, the rest are streamed
    int dev_end(int r_lo, int r_hi) const { return std::max(r_lo, std::min(r_hi, n_dev)); }

    // local rows [r0, r0 + nr) into dst[nr][ld] on the host
    void read(double* dst, const double* dev, int r0, int nr) const
    {
        const int nd = std::max(0, std::min(r0 + nr, n_dev) - r0);
        if (nd > 0) {
            d2h(dst, dev + (size_t)r0 * ld, (size_t)nd * ld * 8);
            dev_sync();
        }
        if (nr > nd) memcpy(dst + (size_t)nd * ld, host_row(r0 + nd), (size_t)(nr - nd) * ld * 8);
    }

#ifndef B200JK_EMULATE
    cudaStream_t copy_stream()     // made on first use, with its events
    {
        if (!cp_stream) {
            CK(cudaStreamCreateWithFlags(&cp_stream, cudaStreamNonBlocking));
            for (cudaEvent_t* e : {&ev_start, &ev_free[0], &ev_free[1]}) CK(cudaEventCreateWithFlags(e, cudaEventDisableTiming));
        }
        return cp_stream;
    }
#endif

    // Visit the local rows [r_lo, r_hi) on the compute stream st: visit(src, r0, nr) once for the rows in HBM, in place (also
    // when the range has no rows at all), then once per block of up to hb host rows staged in d_stage[b & 1].  Blocks 0 and 1 are
    // copied while the device rows are visited, block b + 2 once st is done with block b; the copies follow the work queued on st
    // before the walk.  timed: record the copy and wait events of every block and count the bytes (read_times gives the times).
    template <class F>
    void walk(const double* dev, int r_lo, int r_hi, int hb, bool timed, stream_t st, F visit)
    {
        const int r_dev = dev_end(r_lo, r_hi);
        const int nblk = r_dev < r_hi ? (r_hi - r_dev + hb - 1) / hb : 0;
        if (timed) { bytes = 0; copy_ms = 0.0; exposed_ms = 0.0; timed_blocks = nblk; }
#ifndef B200JK_EMULATE
        if (nblk > 0) {
            copy_stream();
            while (blk_ev.size() < 4 * (size_t)nblk) { cudaEvent_t e; CK(cudaEventCreate(&e)); blk_ev.push_back(e); }
            CK(cudaEventRecord(ev_start, st));
            CK(cudaStreamWaitEvent(cp_stream, ev_start, 0));
        }
#endif
        auto copy = [&](int b) {
            const int a = r_dev + b * hb, nr = std::min(hb, r_hi - a);
#ifndef B200JK_EMULATE
            if (b >= 2) CK(cudaStreamWaitEvent(cp_stream, ev_free[b & 1], 0));
            if (timed) CK(cudaEventRecord(blk_ev[4 * b], cp_stream));
            CK(cudaMemcpyAsync(d_stage[b & 1], host_row(a), (size_t)nr * ld * 8, cudaMemcpyHostToDevice, cp_stream));
            CK(cudaEventRecord(blk_ev[4 * b + 1], cp_stream));
#else
            memcpy(d_stage[b & 1], host_row(a), (size_t)nr * ld * 8);
#endif
        };
        for (int b = 0; b < std::min(nblk, 2); b++) copy(b);
        if (r_dev > r_lo || nblk == 0) visit(dev + (size_t)r_lo * ld, r_lo, r_dev - r_lo);
        for (int b = 0; b < nblk; b++) {
            const int a = r_dev + b * hb, nr = std::min(hb, r_hi - a);
#ifndef B200JK_EMULATE
            if (timed) CK(cudaEventRecord(blk_ev[4 * b + 2], st));
            CK(cudaStreamWaitEvent(st, blk_ev[4 * b + 1], 0));
            if (timed) CK(cudaEventRecord(blk_ev[4 * b + 3], st));
#endif
            visit(d_stage[b & 1], a, nr);
#ifndef B200JK_EMULATE
            CK(cudaEventRecord(ev_free[b & 1], st));
#endif
            if (b + 2 < nblk) copy(b + 2);
            if (timed) bytes += (int64_t)nr * ld * 8;
        }
    }

#ifndef B200JK_EMULATE
    // copy and exposed copy time of the last timed walk, once its stream is synchronised
    void read_times()
    {
        for (int b = 0; b < timed_blocks; b++) {
            float tc = 0, tw = 0;
            CK(cudaEventElapsedTime(&tc, blk_ev[4 * b], blk_ev[4 * b + 1]));
            CK(cudaEventElapsedTime(&tw, blk_ev[4 * b + 2], blk_ev[4 * b + 3]));
            copy_ms += tc; exposed_ms += tw;
        }
    }
#endif
};

// Per-stage device timers: mark(tag) ... mark(-1) brackets one stage with CUDA events on the stream, without host
// synchronisation; read() adds the brackets of each tag in [0, nstage) up into ms (and counts them into n unless it is null)
// once the stream is synchronised.  The emulation has no device time: read() gives zeros.
#ifndef B200JK_EMULATE
struct StageTimer {
    std::vector<cudaEvent_t> ev; std::vector<int> tag; size_t used = 0;
    ~StageTimer() { for (cudaEvent_t e : ev) cudaEventDestroy(e); }
    void start() { used = 0; tag.clear(); }
    void mark(int t, stream_t st)
    {
        if (used == ev.size()) { cudaEvent_t e; CK(cudaEventCreate(&e)); ev.push_back(e); }
        CK(cudaEventRecord(ev[used++], st));
        tag.push_back(t);
    }
    void read(double* ms, int* n, int nstage) const
    {
        for (int i = 0; i < nstage; i++) { ms[i] = 0; if (n) n[i] = 0; }
        for (size_t i = 0; i + 1 < used; i++) {
            if (tag[i] < 0) continue;
            float t = 0;
            CK(cudaEventElapsedTime(&t, ev[i], ev[i + 1]));
            ms[tag[i]] += t;
            if (n) n[tag[i]]++;
        }
    }
};
#else
struct StageTimer {
    void start() {}
    void mark(int, stream_t) {}
    void read(double* ms, int* n, int nstage) const { for (int i = 0; i < nstage; i++) { ms[i] = 0; if (n) n[i] = 0; } }
};
#endif

struct DFState {
    std::vector<DevShell> ash;
    int nash = 0, naux_cart = 0, naux_sph = 0, naux = 0;   // naux = rows of cderi (after lin.dep. removal)
    std::vector<PrimPair> aprims;
    PrimPair* d_aprims = nullptr;
    std::vector<ShellPair> akets[LMAX + 1];
    ShellPair* d_akets[LMAX + 1] = {nullptr};
    int64_t* d_aket_off[LMAX + 1] = {nullptr};   // (P|Q): column offset of each aux shell = its Cartesian offset
    int *d_acart_sh = nullptr, *d_acart_comp = nullptr, *d_asph_sh = nullptr, *d_asph_m = nullptr, *d_ash_l = nullptr,
        *d_ash_cart = nullptr, *d_ash_sph = nullptr;
    int64_t* d_ao_off[NPC] = {nullptr};
    int64_t rowlen = 0;
    int64_t* d_pairoff = nullptr;
    long npair = 0;
    std::vector<int64_t> ao_off_h[NPC];
    // pair screening (b200jk_df_set_pair_tol): a row holds only the ncol packed columns whose device shell pair has a Schwarz
    // bound q >= pair_tol, in ascending packed order; col_of[npair] (-1: dropped) and pk_of[ncol] map between the two layouts.
    // Without screening ncol == npair and there are no maps (d_col_of == nullptr).  The build integrates only the kept shell
    // pairs: kpairs / koff are their per-class lists and Cartesian column offsets (the role of pc[c].d_all / d_ao_off).
    long ncol = 0;
    double pair_tol = 0.0;
    int* d_col_of = nullptr;
    int64_t* d_pk_of = nullptr;
    std::vector<int> col_of_h;
    std::vector<int64_t> pk_of_h;
    bool pair_screened = false;
    ShellPair* d_kpairs[NPC] = {nullptr};
    int64_t* d_koff[NPC] = {nullptr};
    std::vector<int64_t> koff_h[NPC];
    int build_rank = 0, build_world = 1, row0 = 0, nrow = 0;   // rows [row0, row0+nrow) of the tensor live on this rank
    double* d_cderi = nullptr;   // the local rows [0, rows.n_dev)
    RowSplit rows;
    double omega = 0.0;
    // metric factor kept for the integral-direct J (df_jk.get_j): Cholesky L (GPU: column-major lower, emulation: row-major
    // lower) or, when the metric is not positive definite, W = diag(w)^-1/2 V^T [naux, naux_sph] row-major
    double *d_fac = nullptr, *d_W = nullptr;
    double* d_Linv = nullptr;   // L^-1 row-major (integral-direct J: the metric solve as two streaming passes), made on first use
    bool fac_chol = true;
    // raw test build (b200jk_df_set_raw_test): the rows are the bare (P|mu nu), there is no metric factor, and the assembled
    // metric (P|Q) [naux_sph][naux_sph] is kept on the host for b200jk_df_get_metric_test
    bool raw = false;
    std::vector<double> raw_j2c;
    // J/K workspaces
    double *d_dmtril = nullptr, *d_rho = nullptr, *d_vjtril = nullptr, *d_A = nullptr, *d_Y = nullptr, *d_occ = nullptr,
           *d_dm = nullptr, *d_vk = nullptr, *d_vj = nullptr;
    size_t ws_rows = 0, ws_nocc = 0, ws_ndm = 0, ws_occ_ndm = 0;
    int k_mode = 1;      // 0: cuBLAS DGEMM (FP64 pipe), 1: int8 slices on the tensor cores (i8gemm.cuh)
    int k_slices = 7;
    int kb_max = -1, np_max = -1;   // b200jk_df_set_kblock: caps on the rows per K block / resident packed rows (-1: none)
    double* d_Y2 = nullptr; double* d_occT = nullptr; size_t y2_cap = 0, occT_cap = 0;
#ifndef B200JK_EMULATE
    cublasHandle_t cublas = nullptr;
    cusolverDnHandle_t cusolver = nullptr;
    i8g::SliceStack SA, SC, SY, SG;
    int* d_rowexp = nullptr;   // [nrow][nao] exponents of the rows (P, a) of the unpacked tensor (made once, first tensor-core K call)
    float* d_rownorm2 = nullptr;   // [nrow][nao] squared 2-norms of the same rows (exponent bound of Y, fused Y slicing)
    double* d_cmax2 = nullptr;     // device scalar: max squared column norm of the right factor of stage 1
    // int8 slices of the unpacked rows [sa_lo, sa_lo + sa_np) of this rank's range kept resident in SA (as many packed rows as
    // memory permits: all of them when the tensor is small or sharded over enough GPUs); the rest is cut per block into SAt
    bool sa_decided = false; int sa_np = 0, sa_ns = 0, sa_lo = 0, sa_hi = 0;
    i8g::SliceStack SAt;
    StageTimer timer;
#endif
    double stage_ms[B200JK_DF_NSTAGE] = {0}; int stage_n[B200JK_DF_NSTAGE] = {0};
    // MO transforms (df_ao2mo.cuh): device ms of stage 1 and stage 2 and host ms of the last call; test cap on the output band rows
    double ao2mo_ms[3] = {0, 0, 0};
    int ao2mo_tile_rows = -1;
    double* h_pin[2] = {nullptr, nullptr}; size_t pin_cap = 0;   // pinned staging of the output bands, kept between calls
    double mp2_ms[3] = {0, 0, 0};   // DF-MP2 (df_mp2.cuh): device ms of stage 1 and stage 2, host ms of the last call
    double rpa_ms[4] = {0, 0, 0, 0};   // DF-RPA (df_rpa.cuh): device ms of stage 1, the Pi GEMMs, the factorisations; host ms
};

namespace {

void df_free(DFState* d)
{
    if (!d) return;
#ifndef B200JK_EMULATE
    for (double* p : d->h_pin) if (p) cudaFreeHost(p);
#endif
    dev_free(d->d_aprims);
    for (int l = 0; l <= LMAX; l++) { dev_free(d->d_akets[l]); dev_free(d->d_aket_off[l]); }
    dev_free(d->d_acart_sh); dev_free(d->d_acart_comp); dev_free(d->d_asph_sh); dev_free(d->d_asph_m);
    dev_free(d->d_ash_l); dev_free(d->d_ash_cart); dev_free(d->d_ash_sph);
    for (int c = 0; c < NPC; c++) { dev_free(d->d_ao_off[c]); dev_free(d->d_kpairs[c]); dev_free(d->d_koff[c]); }
    dev_free(d->d_col_of); dev_free(d->d_pk_of);
    dev_free(d->d_pairoff); dev_free(d->d_cderi); dev_free(d->d_fac); dev_free(d->d_W); dev_free(d->d_Linv);
    dev_free(d->d_dmtril); dev_free(d->d_rho); dev_free(d->d_vjtril); dev_free(d->d_A); dev_free(d->d_Y); dev_free(d->d_occ);
    dev_free(d->d_dm); dev_free(d->d_vk); dev_free(d->d_vj); dev_free(d->d_Y2); dev_free(d->d_occT);
#ifndef B200JK_EMULATE
    d->SA.release(); d->SAt.release(); d->SC.release(); d->SY.release(); d->SG.release();
    dev_free(d->d_rowexp); dev_free(d->d_rownorm2); dev_free(d->d_cmax2);
    if (d->cublas) cublasDestroy(d->cublas);
    if (d->cusolver) cusolverDnDestroy(d->cusolver);
#endif
    delete d;
}

// ---- transform kernels -------------------------------------------------------------------------
// aux index cart -> sph on whole rows: out[P_sph][col] = sum_c T[m,c] in[cart_off + c][col]
struct AuxC2SFn {
    const double* in; double* out; int64_t rowlen; int nrow_sph;
    const int *sph_sh, *sph_m, *sh_l, *sh_cart, *c2s_off; const double* c2s;
    B2_HD void operator()(long idx) const
    {
        int r = (int)(idx / rowlen);
        int64_t col = idx - (int64_t)r * rowlen;
        int s = sph_sh[r], l = sh_l[s], nc = (l + 1) * (l + 2) / 2;
        const double* T = c2s + c2s_off[l] + sph_m[r] * nc;
        double acc = 0.0;
        for (int c = 0; c < nc; c++) {
            double t = T[c];
            if (t != 0.0) acc += t * in[(int64_t)(sh_cart[s] + c) * rowlen + col];
        }
        out[idx] = acc;
    }
};

// AO pair cart blocks of ONE batch of shell pairs of one class -> packed spherical lower triangle out[r][mu(mu+1)/2+nu].
// in: [nrow, cols] row-major, the Cartesian (a,b) block of pair p starts at column off[p] - col0, element X[b*nca + a].
// One thread per (row, pair, m_a, m_b); every (mu >= nu) element of the packed row is produced by exactly one shell pair
// (elements of shell pairs without surviving primitives are never written: the tensor is zero-filled beforehand).
// npair is the row length of out; with pair screening (col_of != nullptr) the element goes to column col_of[packed index].
struct PairC2SBatchFn {
    const double* in; double* out; int64_t cols, col0; long npair;
    const ShellPair* pairs; const int64_t* off; int np; int la, lb;
    const int *sh_sph, *c2s_off; const double* c2s;
    const int* col_of;
    B2_HD void operator()(long idx) const
    {
        const int nsa = 2 * la + 1, nsb = 2 * lb + 1, nca = (la + 1) * (la + 2) / 2, ncb = (lb + 1) * (lb + 2) / 2;
        const long per_row = (long)np * nsa * nsb;
        const long r = idx / per_row;
        long e = idx - r * per_row;
        const int p = (int)(e / (nsa * nsb));
        e -= (long)p * nsa * nsb;
        const int ma = (int)(e / nsb), mb = (int)(e - (long)ma * nsb);
        const ShellPair& sp = pairs[p];
        const long mu = sh_sph[sp.ish] + ma, nu = sh_sph[sp.jsh] + mb;
        if (sp.ish == sp.jsh && mu < nu) return;
        const double* Ta = c2s + c2s_off[la] + ma * nca;
        const double* Tb = c2s + c2s_off[lb] + mb * ncb;
        const double* X = in + r * cols + (off[p] - col0);
        double acc = 0.0;
        for (int b = 0; b < ncb; b++) {
            const double tb = Tb[b];
            if (tb == 0.0) continue;
            for (int a = 0; a < nca; a++) acc += Ta[a] * tb * X[b * nca + a];
        }
        const long hi = mu >= nu ? mu : nu, lo = mu >= nu ? nu : mu;
        const long t = hi * (hi + 1) / 2 + lo;
        out[r * npair + (col_of ? (long)col_of[t] : t)] = acc;
    }
};

// The same scatter for a Cartesian handle (mol.cart = True): the AO functions are the Cartesian components themselves, so each
// output element is one scaled copy, fab * X[b*nca + a] with fab = fac(la) fac(lb) the s/p factors of make_c2c.  One thread per
// (row, pair, a, b); sh_sph holds the Cartesian AO offset of each device shell in the reference's order.
struct PairCartBatchFn {
    const double* in; double* out; int64_t cols, col0; long npair;
    const ShellPair* pairs; const int64_t* off; int np; int la, lb; double fab;
    const int* sh_sph;
    const int* col_of;
    B2_HD void operator()(long idx) const
    {
        const int nca = (la + 1) * (la + 2) / 2, ncb = (lb + 1) * (lb + 2) / 2;
        const long per_row = (long)np * nca * ncb;
        const long r = idx / per_row;
        long e = idx - r * per_row;
        const int p = (int)(e / (nca * ncb));
        e -= (long)p * nca * ncb;
        const int a = (int)(e / ncb), b = (int)(e - (long)a * ncb);
        const ShellPair& sp = pairs[p];
        const long mu = sh_sph[sp.ish] + a, nu = sh_sph[sp.jsh] + b;
        if (sp.ish == sp.jsh && mu < nu) return;
        const long hi = mu >= nu ? mu : nu, lo = mu >= nu ? nu : mu;
        const long t = hi * (hi + 1) / 2 + lo;
        out[r * npair + (col_of ? (long)col_of[t] : t)] = fab * in[r * cols + (off[p] - col0) + b * nca + a];
    }
};

// dmtril[s][t] = D[mu,nu] + D[nu,mu] (diagonal once)      <- pyscf/df/df_jk.py:329-332
// npair is the row length of out; with pair screening (pk_of != nullptr) column c holds the packed element pk_of[c]
struct DmTrilFn {
    const double* dm; double* out; int nao; long npair; const int64_t* pk_of;
    B2_HD void operator()(long idx) const
    {
        long s = idx / npair, t = idx - s * npair;
        if (pk_of) t = pk_of[t];
        long mu = (long)((sqrt(8.0 * (double)t + 1.0) - 1.0) * 0.5);
        while ((mu + 1) * (mu + 2) / 2 <= t) mu++;
        while (mu * (mu + 1) / 2 > t) mu--;
        long nu = t - mu * (mu + 1) / 2;
        const double* D = dm + s * (long)nao * nao;
        out[idx] = (mu == nu) ? D[mu * nao + mu] : D[mu * nao + nu] + D[nu * nao + mu];
    }
};

// element t (packed index) of a tensor row of length npair: the row itself, or through col_of with 0 for a dropped column
B2_HD double packed_elem(const double* row, const int* col_of, long t)
{
    if (!col_of) return row[t];
    const int c = col_of[t];
    return c >= 0 ? row[c] : 0.0;
}

// unpack rows [r0, r0+nr) of the packed tensor (rows of length npair; col_of: pair-screened rows) into full symmetric nao x nao matrices
struct UnpackFn {
    const double* cderi; double* A; int nao; long npair; long r0; const int* col_of;
    B2_HD void operator()(long idx) const
    {
        long n2 = (long)nao * nao;
        long r = idx / n2, e = idx - r * n2;
        long i = e / nao, j = e - i * nao;
        long mu = i >= j ? i : j, nu = i >= j ? j : i;
        A[idx] = packed_elem(cderi + (r0 + r) * npair, col_of, mu * (mu + 1) / 2 + nu);
    }
};

struct UnpackLongFn {   // G[l][P * ncolp + k] = A_P[l][k] (0 for the pad columns k >= nao) from the packed rows r0 + P: the block as nao long rows
    const double* tril; double* out; int nao; long npair; int r0; long ld; int ncolp; const int* col_of;
    B2_HD void operator()(long idx) const
    {
        long l = idx / ld, e = idx - l * ld;
        long P = e / ncolp, k = e - P * ncolp;
        if (k >= nao) { out[idx] = 0.0; return; }
        long hi = l >= k ? l : k, lo = l >= k ? k : l;
        out[idx] = packed_elem(tril + (r0 + P) * npair, col_of, hi * (hi + 1) / 2 + lo);
    }
};
struct IdentityFn { double* a; int n; B2_HD void operator()(long i) const { a[i * (long)n + i] = 1.0; } };
struct IdentityRowsFn {   // rows [r0, r0 + nrow) of the n x n identity into a zero-filled a[nrow][n]
    double* a; int n, r0;
    B2_HD void operator()(long i) const { a[i * (long)n + r0 + i] = 1.0; }
};
struct GatherRowsFn {   // out[i][j] = X_colmajor[(r0+i), j]
    const double* x; double* out; int n, r0;
    B2_HD void operator()(long idx) const { long i = idx / n, j = idx - i * n; out[idx] = x[(r0 + i) + j * (long)n]; }
};
struct TransposeFn {   // out[c][r] = in[r][c]
    const double* in; double* out; int rows, cols;
    B2_HD void operator()(long idx) const { long r = idx / cols, c = idx - r * cols; out[c * (long)rows + r] = in[idx]; }
};
struct MirrorUpperFn {  // fill the strict lower triangle from the upper one
    double* a; int n;
    B2_HD void operator()(long idx) const { long i = idx / n, j = idx - i * n; if (j < i) a[idx] = a[j * (long)n + i]; }
};

struct UnpackTrilFn {   // vj[s][i][j] from vjtril[s][t] (rows of length npair; col_of: kept columns only, 0 for a dropped pair)
    const double* tril; double* out; int nao; long npair; const int* col_of;
    B2_HD void operator()(long idx) const
    {
        long n2 = (long)nao * nao;
        long s = idx / n2, e = idx - s * n2;
        long i = e / nao, j = e - i * nao;
        long mu = i >= j ? i : j, nu = i >= j ? j : i;
        out[idx] = packed_elem(tril + s * npair, col_of, mu * (mu + 1) / 2 + nu);
    }
};

#ifndef B200JK_EMULATE
// rho[s][P] += sum_{t in segment} cderi[P][t] dmtril[s][t]  — grid (segments, groups of DFJ_R rows, dms).  A thread multiplies ONE
// density element with DFJ_R rows: the tensor streams from HBM once while the density vector comes out of L2 once per DFJ_R rows
// (one row at a time, the L2 -> SM traffic is twice the HBM stream and caps the kernel at ~55 % of the HBM peak).
constexpr int DFJ_R = 8;
__global__ void __launch_bounds__(256) dfj_rho_kernel(const double* __restrict__ cderi, const double* __restrict__ dmtril,
                                                      double* __restrict__ rho, long npair, long r0, long r_end, int naux, long seglen,
                                                      long dstride)   // distance between the density vectors of two DMs
{
    const long rb = r0 + (long)blockIdx.y * DFJ_R;
    const int nr = (int)((r_end - rb < DFJ_R) ? r_end - rb : DFJ_R);
    const int s = blockIdx.z;
    const long t0 = blockIdx.x * seglen;
    const long t1 = (t0 + seglen < npair) ? t0 + seglen : npair;
    const double* row = cderi + rb * npair;
    const double* d = dmtril + (long)s * dstride;
    double acc[DFJ_R];
#pragma unroll
    for (int r = 0; r < DFJ_R; r++) acc[r] = 0.0;
    if (nr == DFJ_R) {
#pragma unroll 2
        for (long t = t0 + threadIdx.x; t < t1; t += 256) {
            const double dv = d[t];
#pragma unroll
            for (int r = 0; r < DFJ_R; r++) acc[r] += __ldcs(row + r * npair + t) * dv;     // streamed once: evict first
        }
    } else {
        for (long t = t0 + threadIdx.x; t < t1; t += 256) {
            const double dv = d[t];
#pragma unroll
            for (int r = 0; r < DFJ_R; r++)
                if (r < nr) acc[r] += __ldcs(row + r * npair + t) * dv;
        }
    }
    __shared__ double part[8][DFJ_R];
#pragma unroll
    for (int r = 0; r < DFJ_R; r++) {
        double a = acc[r];
        for (int o = 16; o > 0; o >>= 1) a += __shfl_xor_sync(0xffffffffu, a, o);
        if ((threadIdx.x & 31) == 0) part[threadIdx.x >> 5][r] = a;
    }
    __syncthreads();
    if (threadIdx.x < nr) {
        double tot = 0.0;
        for (int w = 0; w < 8; w++) tot += part[w][threadIdx.x];
        atomicAdd(&rho[(long)s * naux + rb + threadIdx.x], tot);
    }
}
// vjtril[s][t] += sum_{P in this CTA's row range} rho[s][P] cderi[P][t]  — thread per column, grid (column blocks, row ranges): the
// row ranges make the launch many waves deep (one row range = 1.2 waves on C60: 30 % of the time in a nearly empty second wave)
__global__ void __launch_bounds__(256) dfj_acc_kernel(const double* __restrict__ cderi, const double* __restrict__ rho,
                                                      double* __restrict__ vjtril, long npair, long r0, int nr, int naux, int n_dm,
                                                      long vstride)   // distance between the output vectors of two DMs
{
    long t = blockIdx.x * 256L + threadIdx.x;
    if (t >= npair) return;
    const int per = (nr + gridDim.y - 1) / gridDim.y;
    const int ra = blockIdx.y * per, rb = (ra + per < nr) ? ra + per : nr;
    for (int s = 0; s < n_dm; s++) {
        double a0 = 0.0, a1 = 0.0, a2 = 0.0, a3 = 0.0;
        const double* rh = rho + (long)s * naux + r0;
        const double* col = cderi + r0 * npair + t;
        int r = ra;
        for (; r + 4 <= rb; r += 4) {
            a0 += rh[r] * __ldcs(col + (long)r * npair);
            a1 += rh[r + 1] * __ldcs(col + (long)(r + 1) * npair);
            a2 += rh[r + 2] * __ldcs(col + (long)(r + 2) * npair);
            a3 += rh[r + 3] * __ldcs(col + (long)(r + 3) * npair);
        }
        for (; r < rb; r++) a0 += rh[r] * __ldcs(col + (long)r * npair);
        const double v = (a0 + a1) + (a2 + a3);
        if (gridDim.y == 1) vjtril[(long)s * vstride + t] += v;
        else atomicAdd(&vjtril[(long)s * vstride + t], v);
    }
}
// y[s][r] += sum_c M[r][c] x[s][c]   and   y[s][c] += sum_r M[r][c] x[s][r]   for a row-major M[nrow][ncol]: the two streaming
// kernels above, used by the integral-direct J for its contractions with the 3-center batches and with the metric factor
static void rows_dot(const double* M, long nrow, long ncol, const double* x, long xstride, double* y, int ystride, int n_dm, cudaStream_t st)
{
    const long seglen = 16384;
    const unsigned nseg = (unsigned)((ncol + seglen - 1) / seglen);
    for (long r0 = 0; r0 < nrow; r0 += 32768L * DFJ_R) {
        long nr = std::min<long>(32768L * DFJ_R, nrow - r0);
        dfj_rho_kernel<<<dim3(nseg, (unsigned)((nr + DFJ_R - 1) / DFJ_R), n_dm), 256, 0, st>>>(M, x, y, ncol, r0, r0 + nr, ystride, seglen, xstride);
    }
    CK(cudaGetLastError());
}
static void cols_acc(const double* M, long nrow, long ncol, const double* x, int xstride, double* y, long ystride, int n_dm, cudaStream_t st)
{
    const unsigned ncb = (unsigned)((ncol + 255) / 256);
    unsigned gy = (unsigned)std::max<long>(1, std::min<long>(nrow / 64, (6L * device_sm_count() * 8 + ncb - 1) / ncb));
    dfj_acc_kernel<<<dim3(ncb, gy), 256, 0, st>>>(M, x, y, ncol, 0, (int)nrow, xstride, n_dm, ystride);
    CK(cudaGetLastError());
}
#endif

// functions per shell in the handle's AO convention: 2l+1 real spherical harmonics, or the ncart(l) Cartesian components of a
// Cartesian handle (the auxiliary basis follows the same convention, as the reference's make_auxmol copies mol.cart)
static int nfun(b200jk_handle h, int l) { return h->cart ? ncart(l) : 2 * l + 1; }

// Auxiliary tables: for a Cartesian handle the "spherical" auxiliary index (naux_sph, d_asph_*) is the Cartesian one in the
// reference's order, and h->d_c2s holds the make_c2c tables, so AuxC2SFn / Cart2SphFn reduce to the s/p factors.
void build_aux(b200jk_handle h, DFState* d, const int32_t* atm, const int32_t* bas, int nbas, const double* env)
{
    std::vector<DevShell> tmp;
    int sph = 0;
    for (int ib = 0; ib < nbas; ib++) {
        const int32_t* b = bas + ib * BAS_SLOTS;
        int l = b[ANG_OF], np = b[NPRIM_OF], nc = b[NCTR_OF];
        if (l > LMAX) throw std::runtime_error("auxiliary angular momentum > g is not supported");
        const double* r = env + atm[b[ATOM_OF] * ATM_SLOTS + PTR_COORD];
        for (int c = 0; c < nc; c++) {
            DevShell s;
            s.l = l; s.ref_shell = ib; s.sph_off = sph + c * nfun(h, l); s.cart_off = 0;
            s.r[0] = r[0]; s.r[1] = r[1]; s.r[2] = r[2];
            for (int p = 0; p < np; p++) {
                double cf = env[b[PTR_COEFF] + c * np + p];
                if (cf != 0.0) { s.e.push_back(env[b[PTR_EXP] + p]); s.c.push_back(cf); }
            }
            s.nprim = (int)s.e.size();
            tmp.push_back(s);
        }
        sph += nc * nfun(h, l);
    }
    d->naux_sph = sph;
    std::stable_sort(tmp.begin(), tmp.end(), [](const DevShell& a, const DevShell& b) { return a.l < b.l; });
    int co = 0;
    for (auto& s : tmp) { s.cart_off = co; co += ncart(s.l); }
    d->naux_cart = co;
    d->ash = tmp;
    d->nash = (int)tmp.size();
    std::vector<int> cart_sh(co), cart_comp(co), sph_sh(sph), sph_m(sph), sh_l(d->nash), sh_cart(d->nash), sh_sph(d->nash);
    std::vector<int64_t> koff[LMAX + 1];
    for (int i = 0; i < d->nash; i++) {
        const DevShell& s = d->ash[i];
        sh_l[i] = s.l; sh_cart[i] = s.cart_off; sh_sph[i] = s.sph_off;
        for (int a = 0; a < ncart(s.l); a++) { cart_sh[s.cart_off + a] = i; cart_comp[s.cart_off + a] = a; }
        for (int m = 0; m < nfun(h, s.l); m++) { sph_sh[s.sph_off + m] = i; sph_m[s.sph_off + m] = m; }
        ShellPair sp{};
        sp.ish = i; sp.jsh = -1; sp.i0 = s.cart_off; sp.j0 = 0; sp.same = 0;
        sp.prim_off = (int)d->aprims.size(); sp.nprim = s.nprim;
        for (int p = 0; p < s.nprim; p++) {
            PrimPair pp;
            pp.p = s.e[p]; pp.Px = s.r[0]; pp.Py = s.r[1]; pp.Pz = s.r[2];
            pp.PAx = pp.PAy = pp.PAz = 0.0;
            pp.cc = s.c[p] / s.e[p] * 5.914967172795612486;
            d->aprims.push_back(pp);
        }
        d->akets[s.l].push_back(sp);
        koff[s.l].push_back(s.cart_off);
    }
    d->d_aprims = upload(d->aprims);
    for (int l = 0; l <= LMAX; l++) { d->d_akets[l] = upload(d->akets[l]); d->d_aket_off[l] = upload(koff[l]); }
    d->d_acart_sh = upload(cart_sh); d->d_acart_comp = upload(cart_comp); d->d_asph_sh = upload(sph_sh); d->d_asph_m = upload(sph_m);
    d->d_ash_l = upload(sh_l); d->d_ash_cart = upload(sh_cart); d->d_ash_sph = upload(sh_sph);
}

#ifdef B200JK_EMULATE
// tiny dense helpers for the CPU emulation (tests only)
void cpu_cholesky_lower(std::vector<double>& a, int n, bool& ok)
{   // row-major symmetric -> L in lower triangle
    ok = true;
    for (int j = 0; j < n; j++) {
        double s = a[(size_t)j * n + j];
        for (int k = 0; k < j; k++) s -= a[(size_t)j * n + k] * a[(size_t)j * n + k];
        if (!(s > 0)) { ok = false; return; }
        double ljj = std::sqrt(s);
        a[(size_t)j * n + j] = ljj;
        for (int i = j + 1; i < n; i++) {
            double t = a[(size_t)i * n + j];
            for (int k = 0; k < j; k++) t -= a[(size_t)i * n + k] * a[(size_t)j * n + k];
            a[(size_t)i * n + j] = t / ljj;
        }
    }
}
#endif

}  // namespace

// ------------------------------------------------------------------------------------------------
// (ij|P) for all AO shell pairs in batches of bounded scratch: Cartesian rows d_xc[naux_cart, cols] -> spherical aux rows
// d_xa[naux_sph, cols]; use(col0, cols) consumes one batch (columns = Cartesian pair blocks, DFState::ao_off_h).
// kept: only the shell pairs that survive pair screening (DFState::kpairs / koff_h), else all of them.
template <class F>
static void for_each_j3c_batch(b200jk_handle h, DFState* d, double omega, stream_t st, F use, bool kept = false)
{
    const int nac = d->naux_cart, nas = d->naux_sph;
    const int64_t budget_cols = std::max<int64_t>(4096, (int64_t)((3ULL << 30) / ((size_t)nac * 8)));
    double* d_xc = (double*)dev_alloc((size_t)nac * (size_t)std::min<int64_t>(budget_cols + 128, d->rowlen) * 8);
    double* d_xa = (double*)dev_alloc((size_t)nas * (size_t)std::min<int64_t>(budget_cols + 128, d->rowlen) * 8);
    for (int cb = 0; cb < NPC; cb++) {
        const auto& offs = kept ? d->koff_h[cb] : d->ao_off_h[cb];
        const ShellPair* pairs = kept ? d->d_kpairs[cb] : h->pc[cb].d_all;
        const int64_t* d_off = kept ? d->d_koff[cb] : d->d_ao_off[cb];
        const int np_all = (int)offs.size();
        if (np_all == 0) continue;
        const int64_t blk = (int64_t)ncart(h->pc[cb].la) * ncart(h->pc[cb].lb);
        int p0 = 0;
        while (p0 < np_all) {
            int p1 = (int)std::min<int64_t>(np_all, p0 + std::max<int64_t>(1, budget_cols / blk));
            const int64_t col0 = offs[p0], cols = (int64_t)(p1 - p0) * blk;
            for (int lk = 0; lk <= LMAX; lk++) {
                if (d->akets[lk].empty()) continue;
                J3cParams P{};
                P.bra_pairs = pairs + p0; P.nbra = p1 - p0; P.bra_out_off = d_off + p0;
                P.ket_shells = d->d_akets[lk]; P.nket = (int)d->akets[lk].size();
                P.bra_prims = h->d_prims; P.ket_prims = d->d_aprims;
                P.tb = h->tb; P.omega = omega; P.out = d_xc; P.row_stride = cols; P.col0 = col0;
                launch_j3c(cb, lk, P, st);
            }
            AuxC2SFn a2 {d_xc, d_xa, cols, nas, d->d_asph_sh, d->d_asph_m, d->d_ash_l, d->d_ash_cart, h->d_c2s_off, h->d_c2s};
            launch_1d((long)nas * cols, a2, st);
            use(col0, cols, d_xa, cb, p0, p1);
            p0 = p1;
        }
    }
#ifndef B200JK_EMULATE
    CK(cudaStreamSynchronize(st));
#endif
    dev_free(d_xc); dev_free(d_xa);
}

// Pair screening of the tensor's columns: the Schwarz bound q = sqrt((ab|ab)) of every device shell pair for the tensor's own
// operator (SchwarzSphFn: the reference's normalisation, per segment of a general contraction, as b200jk_set_screening computes
// it, but on a copy of the pair list so that the 4-center screening state of the handle is left as it is).  A packed column
// (mu >= nu) is kept iff the q of its shell pair is >= tol; ||B[:, mu nu]||_2^2 = (mu nu|P) M^-1 (P|mu nu) <= (mu nu|mu nu)
// bounds a dropped column by q < tol.  Shell pairs without a surviving primitive pair are not in pc[c].all: always dropped.
// Fills ncol, col_of / pk_of (host and device) and the per-class kept pair lists with their Cartesian column offsets.
static void select_pairs(b200jk_handle h, DFState* d, double omega, double tol, stream_t st)
{
    const long npair = d->npair;
    std::vector<char> keep((size_t)npair, 0);
    int64_t off = 0;
    for (int c = 0; c < NPC; c++) {
        PairClass& P = h->pc[c];
        std::vector<ShellPair> pairs = P.all;
        std::vector<int64_t> koff;
        if (!pairs.empty()) {
            ShellPair* d_tmp = upload(pairs);
            const long ne = (long)ncart(P.la) * ncart(P.lb);
            const long chunk = std::max<long>(1, (256L << 20) / (ne * ne * 8));     // <= 256 MB of scratch per launch
            double* scratch = (double*)dev_alloc((size_t)std::min<long>(chunk, (long)pairs.size()) * ne * ne * 8);
            for (long i0 = 0; i0 < (long)pairs.size(); i0 += chunk) {
                const long n = std::min<long>(chunk, (long)pairs.size() - i0);
                SchwarzSphFn fn{d_tmp + i0, h->d_prims, h->tb, omega, P.la, P.lb, h->d_c2s + h->c2s_off[P.la], h->d_c2s + h->c2s_off[P.lb],
                                scratch, nfun(h, P.la), nfun(h, P.lb)};
                launch_1d(n, fn, st);
#ifndef B200JK_EMULATE
                CK(cudaStreamSynchronize(st));
#endif
            }
            d2h(pairs.data(), d_tmp, pairs.size() * sizeof(ShellPair), st);
#ifndef B200JK_EMULATE
            CK(cudaStreamSynchronize(st));
#endif
            dev_free(scratch); dev_free(d_tmp);
        }
        std::vector<ShellPair> kept;
        for (const ShellPair& sp : pairs) {
            if (!(sp.q >= tol)) continue;
            kept.push_back(sp);
            koff.push_back(off);
            off += ncart(P.la) * ncart(P.lb);
            const DevShell &a = h->sh[sp.ish], &b = h->sh[sp.jsh];
            for (int ma = 0; ma < nfun(h, a.l); ma++)
                for (int mb = 0; mb < nfun(h, b.l); mb++) {
                    const long mu = a.sph_off + ma, nu = b.sph_off + mb;
                    if (sp.ish == sp.jsh && mu < nu) continue;
                    const long hi = std::max(mu, nu), lo = std::min(mu, nu);
                    keep[(size_t)(hi * (hi + 1) / 2 + lo)] = 1;
                }
        }
        d->d_kpairs[c] = upload(kept);
        d->d_koff[c] = upload(koff);
        d->koff_h[c] = koff;
    }
    d->col_of_h.assign((size_t)npair, -1);
    d->pk_of_h.clear();
    for (long t = 0; t < npair; t++)
        if (keep[(size_t)t]) { d->col_of_h[(size_t)t] = (int)d->pk_of_h.size(); d->pk_of_h.push_back(t); }
    d->ncol = (long)d->pk_of_h.size();
    if (d->ncol == 0) throw std::runtime_error("pair screening: no AO-pair column has a Schwarz bound >= pair_tol");
    d->d_col_of = upload(d->col_of_h);
    d->d_pk_of = upload(d->pk_of_h);
    d->pair_screened = true;
    d->pair_tol = tol;
}

static int df_build_impl(b200jk_handle h, const int32_t* aux_atm, int aux_natm, const int32_t* aux_bas, int aux_nbas,
                         const double* aux_env, int aux_nenv, double omega, double lindep, bool j_only)
{
    if (!h) return 1;
    try {
        (void)aux_natm; (void)aux_nenv;
        if (h->df) { df_free(h->df); h->df = nullptr; }
        DFState* d = new DFState();
        h->df = d; h->df_free = df_free;
        d->omega = omega;
#ifndef B200JK_EMULATE
        CK(cudaSetDevice(h->device));
        cudaStream_t st = h->stream;
        CKB(cublasCreate(&d->cublas));
        CKS(cusolverDnCreate(&d->cusolver));
#else
        stream_t st = 0;
#endif
        build_aux(h, d, aux_atm, aux_bas, aux_nbas, aux_env);
        const int nao = h->nsph, nsh = h->nsh;
        d->npair = (long)nao * (nao + 1) / 2;

        // ---- row layout of the Cartesian (ij| blocks and the (shell,shell) -> offset table
        std::vector<int64_t> pairoff((size_t)nsh * nsh, -1);
        int64_t off = 0;
        for (int c = 0; c < NPC; c++) {
            std::vector<int64_t> o;
            for (auto& sp : h->pc[c].all) {
                o.push_back(off);
                pairoff[(size_t)sp.ish * nsh + sp.jsh] = off;
                off += (int64_t)ncart(h->pc[c].la) * ncart(h->pc[c].lb);
            }
            d->d_ao_off[c] = upload(o);
            d->ao_off_h[c] = o;
        }
        d->rowlen = off;
        d->d_pairoff = upload(pairoff);
        d->ncol = d->npair;
        if (!j_only && h->df_pair_tol > 0.0) select_pairs(h, d, omega, h->df_pair_tol, st);

        // ---- (P|Q) in the Cartesian aux basis, then to spherical
        const int nac = d->naux_cart, nas = d->naux_sph;
        double* d_j2c_cart = (double*)dev_alloc((size_t)nac * nac * 8);
        dev_zero(d_j2c_cart, (size_t)nac * nac * 8, st);
        for (int lp = 0; lp <= LMAX; lp++)
            for (int lq = 0; lq <= LMAX; lq++) {
                if (d->akets[lp].empty() || d->akets[lq].empty()) continue;
                J3cParams P{};
                P.bra_pairs = d->d_akets[lp]; P.nbra = (int)d->akets[lp].size(); P.bra_out_off = d->d_aket_off[lp];
                P.ket_shells = d->d_akets[lq]; P.nket = (int)d->akets[lq].size();
                P.bra_prims = d->d_aprims; P.ket_prims = d->d_aprims;
                P.tb = h->tb; P.omega = omega; P.out = d_j2c_cart; P.row_stride = nac;
                int cb = (lp == 4) ? 10 : pair_class_id(lp, 0);
                launch_j3c(cb, lq, P, st);
            }
        double* d_j2c = (double*)dev_alloc((size_t)nas * nas * 8);
        Cart2SphFn c2 {d_j2c_cart, d_j2c, nas, nac, 0.0, 0, d->d_asph_sh, d->d_asph_m, d->d_ash_l, d->d_ash_cart, h->d_c2s_off, h->d_c2s};
        launch_1d((long)nas * nas, c2, st);

        // ---- metric decomposition: Cholesky, or eigendecomposition when it is not positive definite
        //      (incore.py:150-158; _eig_decompose :263-270 keeps w > lindep)
        bool use_chol = true;
        std::vector<double> W;   // eig fallback: [naux_kept, naux] row-major
        int nkeep = nas;
        // raw test build: keep (P|Q), skip the factorisation (the erf metric need not be positive definite) and use the identity
        // as the metric transform below, so that the rows are the bare 3-center integrals
        const bool raw = h->df_raw_test && !j_only;
        if (raw) {
            d->raw = true;
            d->raw_j2c.resize((size_t)nas * nas);
            d2h(d->raw_j2c.data(), d_j2c, (size_t)nas * nas * 8, st);
#ifndef B200JK_EMULATE
            CK(cudaStreamSynchronize(st));
#endif
        }
#ifndef B200JK_EMULATE
        if (!raw) {
            int lwork = 0;
            CKS(cusolverDnSetStream(d->cusolver, st));
            CKB(cublasSetStream(d->cublas, st));
            double* d_chol = (double*)dev_alloc((size_t)nas * nas * 8);
            CK(cudaMemcpyAsync(d_chol, d_j2c, (size_t)nas * nas * 8, cudaMemcpyDeviceToDevice, st));
            CKS(cusolverDnDpotrf_bufferSize(d->cusolver, CUBLAS_FILL_MODE_LOWER, nas, d_chol, nas, &lwork));
            double* d_work = (double*)dev_alloc((size_t)lwork * 8);
            int* d_info = (int*)dev_alloc(4);
            CKS(cusolverDnDpotrf(d->cusolver, CUBLAS_FILL_MODE_LOWER, nas, d_chol, nas, d_work, lwork, d_info));
            int info = 0;
            d2h(&info, d_info, 4, st);
            CK(cudaStreamSynchronize(st));
            dev_free(d_work);
            if (info != 0) {
                use_chol = false;
                // eigendecomposition on device
                double* d_w = (double*)dev_alloc((size_t)nas * 8);
                CK(cudaMemcpyAsync(d_chol, d_j2c, (size_t)nas * nas * 8, cudaMemcpyDeviceToDevice, st));
                CKS(cusolverDnDsyevd_bufferSize(d->cusolver, CUSOLVER_EIG_MODE_VECTOR, CUBLAS_FILL_MODE_LOWER, nas, d_chol, nas, d_w, &lwork));
                d_work = (double*)dev_alloc((size_t)lwork * 8);
                CKS(cusolverDnDsyevd(d->cusolver, CUSOLVER_EIG_MODE_VECTOR, CUBLAS_FILL_MODE_LOWER, nas, d_chol, nas, d_w, d_work, lwork, d_info));
                std::vector<double> w(nas), V((size_t)nas * nas);
                d2h(w.data(), d_w, (size_t)nas * 8, st);
                d2h(V.data(), d_chol, (size_t)nas * nas * 8, st);   // column-major eigenvectors: V[i + j*n]
                CK(cudaStreamSynchronize(st));
                dev_free(d_work); dev_free(d_w);
                nkeep = 0;
                for (int j = 0; j < nas; j++) if (w[j] > lindep) nkeep++;
                W.assign((size_t)nkeep * nas, 0.0);
                int k = 0;
                for (int j = 0; j < nas; j++) {
                    if (!(w[j] > lindep)) continue;
                    double sc = 1.0 / std::sqrt(w[j]);
                    for (int i = 0; i < nas; i++) W[(size_t)k * nas + i] = V[(size_t)i + (size_t)j * nas] * sc;
                    k++;
                }
            }
            dev_free(d_info);
            // keep the factor in d_j2c (column-major lower == row-major upper of the same symmetric storage)
            if (use_chol) CK(cudaMemcpyAsync(d_j2c, d_chol, (size_t)nas * nas * 8, cudaMemcpyDeviceToDevice, st));
            else { d->d_W = (double*)dev_alloc((size_t)std::max(nkeep, 1) * nas * 8); h2d(d->d_W, W.data(), (size_t)nkeep * nas * 8, st); CK(cudaStreamSynchronize(st)); }
            dev_free(d_chol);
        }
#else
        std::vector<double> j2c_h((size_t)nas * nas);
        d2h(j2c_h.data(), d_j2c, (size_t)nas * nas * 8);
        if (!raw) {
            std::vector<double> Lm = j2c_h;
            bool ok;
            cpu_cholesky_lower(Lm, nas, ok);
            if (!ok) throw std::runtime_error("emulation: metric not positive definite (eig fallback is GPU-only)");
            j2c_h = Lm;
            memcpy(d_j2c, Lm.data(), (size_t)nas * nas * 8);   // emulation: row-major lower factor
        }
        (void)lindep;
#endif
        d->naux = nkeep;
        d->fac_chol = use_chol;
        if (raw) dev_free(d_j2c);
        else d->d_fac = d_j2c;
        if (j_only) {   // integral-direct J only (b200jk_df_prepare_j): no tensor
#ifndef B200JK_EMULATE
            CK(cudaStreamSynchronize(st));
#endif
            dev_free(d_j2c_cart);
            d->row0 = 0; d->nrow = 0;
            return 0;
        }

        // ---- rows of the metric transform owned by this rank: T[nloc][nas] (rows of L^-1, or of W = diag(w)^-1/2 V^T)
        const int bw = h->shard_world, br = h->shard_rank;
        int r_lo, r_hi;
        shard_range(nkeep, br, bw, r_lo, r_hi);
        const int nloc = r_hi - r_lo;
        d->build_rank = br; d->build_world = bw; d->row0 = r_lo; d->nrow = nloc;
        double* d_T = (double*)dev_alloc((size_t)std::max(nloc, 1) * nas * 8);
        if (raw) {
            dev_zero(d_T, (size_t)std::max(nloc, 1) * nas * 8, st);
            IdentityRowsFn idr{d_T, nas, r_lo};
            launch_1d(nloc, idr, st);
        }
#ifndef B200JK_EMULATE
        else if (use_chol) {
            // L^-1 by one triangular solve against the identity (naux^2, setup only), then gather this rank's rows
            double* d_inv = (double*)dev_alloc((size_t)nas * nas * 8);
            dev_zero(d_inv, (size_t)nas * nas * 8, st);
            IdentityFn idf{d_inv, nas};
            launch_1d(nas, idf, st);
            const double one = 1.0;
            CKB(cublasDtrsm(d->cublas, CUBLAS_SIDE_LEFT, CUBLAS_FILL_MODE_LOWER, CUBLAS_OP_N, CUBLAS_DIAG_NON_UNIT, nas, nas, &one, d_j2c, nas,
                            d_inv, nas));
            GatherRowsFn gf{d_inv, d_T, nas, r_lo};   // d_inv is column-major: X[(i) + j*n]
            launch_1d((long)nloc * nas, gf, st);
            CK(cudaStreamSynchronize(st));
            dev_free(d_inv);
        } else {
            h2d(d_T, W.data() + (size_t)r_lo * nas, (size_t)nloc * nas * 8, st);
        }
#else
        else {   // host: rows of L^-1 by forward substitution on unit vectors (tests only)
            std::vector<double> inv((size_t)nas * nas, 0.0);
            for (int c = 0; c < nas; c++) {
                for (int i = c; i < nas; i++) {
                    double sacc = (i == c) ? 1.0 : 0.0;
                    for (int k = c; k < i; k++) sacc -= j2c_h[(size_t)i * nas + k] * inv[(size_t)k * nas + c];
                    inv[(size_t)i * nas + c] = sacc / j2c_h[(size_t)i * nas + i];
                }
            }
            memcpy(d_T, inv.data() + (size_t)r_lo * nas, (size_t)nloc * nas * 8);
        }
#endif

        // ---- (ij|P) in batches of AO shell pairs (bounded scratch): Cartesian rows -> spherical aux -> T . (P|ij) -> packed
        //      spherical columns of this batch.  Nothing of size naux x (all Cartesian pairs) ever exists: the largest buffers are
        //      the tensor itself and three batch-sized scratch arrays (<= ~3 GB each), so a 111 GB tensor fits one 180 GB GPU.
        const long ncol = d->ncol;   // row length: every packed column, or the kept ones under pair screening
        const int64_t bcols = std::min<int64_t>(std::max<int64_t>(4096, (int64_t)((3ULL << 30) / ((size_t)d->naux_cart * 8))) + 128, d->rowlen);
        double* d_ybatch = (double*)dev_alloc((size_t)std::max(nloc, 1) * (size_t)bcols * 8);
        const std::string split_err = d->rows.plan(h, nloc, ncol, d->k_slices, true, &d->d_cderi, st);
        if (!split_err.empty()) {
            dev_free(d_T); dev_free(d_ybatch); dev_free(d_j2c_cart);
            df_free(d); h->df = nullptr;
            throw std::runtime_error(split_err);
        }
        const int n_dev = d->rows.n_dev, n_host = nloc - n_dev;
        // rows of the tensor from the rows Trows[nr][nas] of the metric transform into out[nr][ncol] (zero-filled); under pair
        // screening only the kept shell pairs are integrated and their columns written through col_of
        const bool kept = d->pair_screened;
        auto fill_rows = [&](const double* Trows, int nr, double* out) {
            for_each_j3c_batch(h, d, omega, st, [&](int64_t col0, int64_t cols, const double* d_xa, int cb, int p0, int p1) {
                if (nr <= 0) return;
                if (cols > bcols) throw std::runtime_error("internal: 3-center batch larger than its scratch buffer");
#ifndef B200JK_EMULATE
                // row-major Y[nr, cols] = T[nr, nas] . Xa[nas, cols]  <=>  col-major Y^T = Xa^T . T^T
                const double one = 1.0, zero = 0.0;
                CKB(cublasDgemm(d->cublas, CUBLAS_OP_N, CUBLAS_OP_N, (int)cols, nr, nas, &one, d_xa, (int)cols, Trows, nas, &zero,
                                d_ybatch, (int)cols));
#else
                for (int i = 0; i < nr; i++)
                    for (int64_t c = 0; c < cols; c++) {
                        double acc = 0.0;
                        for (int k = 0; k < nas; k++) acc += Trows[(size_t)i * nas + k] * d_xa[(size_t)k * cols + c];
                        d_ybatch[(size_t)i * cols + c] = acc;
                    }
#endif
                const int la = h->pc[cb].la, lb = h->pc[cb].lb;
                const ShellPair* bpairs = (kept ? d->d_kpairs[cb] : h->pc[cb].d_all) + p0;
                const int64_t* boff = (kept ? d->d_koff[cb] : d->d_ao_off[cb]) + p0;
                if (h->cart) {
                    PairCartBatchFn p2{d_ybatch, out, cols, col0, ncol, bpairs, boff, p1 - p0, la, lb,
                                       make_c2c(la)[0] * make_c2c(lb)[0], h->d_sh_sph, d->d_col_of};
                    launch_1d((long)nr * (p1 - p0) * ncart(la) * ncart(lb), p2, st);
                } else {
                    PairC2SBatchFn p2{d_ybatch, out, cols, col0, ncol, bpairs, boff, p1 - p0, la, lb, h->d_sh_sph, h->d_c2s_off, h->d_c2s,
                                      d->d_col_of};
                    launch_1d((long)nr * (p1 - p0) * (2 * la + 1) * (2 * lb + 1), p2, st);
                }
            }, kept);
        };
        if (n_dev > 0 || n_host == 0) fill_rows(d_T, n_dev, d->d_cderi);
        if (n_host > 0) {
            // host rows in blocks as large as the device memory left over allows (the K reserve is not in use yet); the 3-center
            // integrals are recomputed once per block (d_ybatch holds nloc >= hb rows)
            long hb = d->rows.stage_rows;
#ifndef B200JK_EMULATE
            size_t freeb = 0, totb = 0;
            CK(cudaMemGetInfo(&freeb, &totb));
            const double scratch = (double)(d->naux_cart + nas) * bcols * 8 + (double)(1UL << 30);   // for_each_j3c_batch + margin
            if ((double)freeb > scratch + ncol * 8.0) hb = std::max(hb, (long)(((double)freeb - scratch) / (ncol * 8.0)));
#endif
            hb = std::max(1L, std::min<long>(hb, n_host));
            double* d_blk = (double*)dev_alloc((size_t)hb * ncol * 8);
            for (int a = n_dev; a < nloc; a += (int)hb) {
                const int nr = (int)std::min<long>(hb, nloc - a);
                dev_zero(d_blk, (size_t)nr * ncol * 8, st);
                fill_rows(d_T + (size_t)a * nas, nr, d_blk);
                d2h(d->rows.host_row(a), d_blk, (size_t)nr * ncol * 8, st);
            }
#ifndef B200JK_EMULATE
            CK(cudaStreamSynchronize(st));
#endif
            dev_free(d_blk);
        }
        dev_free(d_T);
        dev_free(d_ybatch);
#ifndef B200JK_EMULATE
        CK(cudaStreamSynchronize(st));
#endif
        dev_free(d_j2c_cart);
    } catch (std::exception& e) { set_err(h, e.what()); return 2; }
    return 0;
}

extern "C" int b200jk_df_build(b200jk_handle h, const int32_t* aux_atm, int aux_natm, const int32_t* aux_bas, int aux_nbas,
                               const double* aux_env, int aux_nenv, double omega, double lindep)
{
    return df_build_impl(h, aux_atm, aux_natm, aux_bas, aux_nbas, aux_env, aux_nenv, omega, lindep, false);
}

// Integral-direct DF-J without the tensor (df_jk.get_j, pyscf/df/df_jk.py:415-506): prepare = auxiliary tables + metric
// factor (the reference's cached dfobj._vjopt with its cho_factor'ed j2c) ...
extern "C" int b200jk_df_prepare_j(b200jk_handle h, const int32_t* aux_atm, int aux_natm, const int32_t* aux_bas, int aux_nbas,
                                   const double* aux_env, int aux_nenv, double omega, double lindep)
{
    return df_build_impl(h, aux_atm, aux_natm, aux_bas, aux_nbas, aux_env, aux_nenv, omega, lindep, true);
}

namespace {
// Dc[s][off + b*NI + a] = D_cart[i0+a][j0+b] (+ transpose element for off-diagonal shell pairs; D_cart is symmetric)
struct PairGatherFn {
    const ShellPair* pairs; const int64_t* off; int ni, nj, ncart_; const double* dcart; double* dc; int64_t rowlen;
    B2_HD void operator()(long idx) const
    {
        const int blk = ni * nj;
        long s = idx / ((long)npairs * blk), r = idx - s * (long)npairs * blk;
        long p = r / blk; int e = (int)(r - p * blk);
        int b = e / ni, a = e - b * ni;
        const ShellPair& sp = pairs[p];
        double v = dcart[(size_t)s * ncart_ * ncart_ + (size_t)(sp.i0 + a) * ncart_ + sp.j0 + b];
        dc[(size_t)s * rowlen + off[p] + e] = (sp.ish == sp.jsh) ? v : 2.0 * v;
    }
    int npairs;
};
// Jacc_cart[s][i0+a][j0+b] = w Jc[s][off + b*NI + a], w = 1/2 on diagonal shell pairs (J = Jacc + Jacc^T afterwards)
struct PairScatterFn {
    const ShellPair* pairs; const int64_t* off; int ni, nj, ncart_; const double* jc; double* jcart; int64_t rowlen; int npairs;
    B2_HD void operator()(long idx) const
    {
        const int blk = ni * nj;
        long s = idx / ((long)npairs * blk), r = idx - s * (long)npairs * blk;
        long p = r / blk; int e = (int)(r - p * blk);
        int b = e / ni, a = e - b * ni;
        const ShellPair& sp = pairs[p];
        double v = jc[(size_t)s * rowlen + off[p] + e];
        jcart[(size_t)s * ncart_ * ncart_ + (size_t)(sp.i0 + a) * ncart_ + sp.j0 + b] = (sp.ish == sp.jsh) ? 0.5 * v : v;
    }
};
}  // namespace

// ... and the two passes over the 3-center integrals:  rho = j2c^-1 (P|ij) D_ji ,  J_ij = (ij|P) rho_P
extern "C" int b200jk_df_direct_j(b200jk_handle h, const double* dm, int n_dm, int nao, double* vj)
{
    if (!h) return 1;
    try {
        DFState* d = h->df;
        if (d && d->raw) throw std::runtime_error("b200jk_df_direct_j: a raw test build (b200jk_df_set_raw_test) has no metric factor");
        if (!d || !d->d_fac) throw std::runtime_error("call b200jk_df_prepare_j (or b200jk_df_build) before b200jk_df_direct_j");
        if (nao != h->nsph) throw std::runtime_error("nao does not match the basis of this handle");
        if (n_dm < 1 || !dm || !vj) throw std::runtime_error("bad arguments");
        auto t0 = std::chrono::steady_clock::now();
#ifndef B200JK_EMULATE
        CK(cudaSetDevice(h->device));
        cudaStream_t st = h->stream;
        CKB(cublasSetStream(d->cublas, st));
        CKS(cusolverDnSetStream(d->cusolver, st));
#else
        stream_t st = 0;
#endif
        const int nas = d->naux_sph, nc = h->ncart, ns = h->nsph;
        const size_t ns2 = (size_t)ns * ns, nc2 = (size_t)nc * nc;
        double* d_dsph = (double*)dev_alloc(ns2 * n_dm * 8);
        double* d_dcart = (double*)dev_alloc(nc2 * n_dm * 8);
        double* d_dc = (double*)dev_alloc((size_t)d->rowlen * n_dm * 8);
        double* d_rho = (double*)dev_alloc((size_t)nas * n_dm * 8);
        h2d(d_dsph, dm, ns2 * n_dm * 8, st);
        Sph2CartFn s2c{d_dsph, d_dcart, ns, nc, 0, h->d_cart_sh, h->d_cart_comp, h->d_sh_l, h->d_sh_sph, h->d_c2s_off, h->d_c2s, h->cart};
        launch_1d((long)nc2 * n_dm, s2c, st);
        for (int cb = 0; cb < NPC; cb++) {
            const int np = (int)h->pc[cb].all.size();
            if (!np) continue;
            PairGatherFn g{h->pc[cb].d_all, d->d_ao_off[cb], ncart(h->pc[cb].la), ncart(h->pc[cb].lb), nc, d_dcart, d_dc, d->rowlen, np};
            launch_1d((long)n_dm * np * g.ni * g.nj, g, st);
        }
        dev_zero(d_rho, (size_t)nas * n_dm * 8, st);
        // ---- pass 1: rho[s][P] = sum_col (P|col) Dc[s][col]
        for_each_j3c_batch(h, d, d->omega, st, [&](int64_t col0, int64_t cols, const double* d_xa, int, int, int) {
#ifndef B200JK_EMULATE
            rows_dot(d_xa, nas, cols, d_dc + col0, d->rowlen, d_rho, nas, n_dm, st);
#else
            for (int s = 0; s < n_dm; s++)
                for (int P = 0; P < nas; P++) {
                    double acc = 0.0;
                    for (int64_t c = 0; c < cols; c++) acc += d_xa[(size_t)P * cols + c] * d_dc[(size_t)s * d->rowlen + col0 + c];
                    d_rho[(size_t)s * nas + P] += acc;
                }
#endif
        });
        // ---- solve the metric equation  (cho_solve / the eigen-decomposed inverse)
#ifndef B200JK_EMULATE
        {
            // rho <- F^T (F rho) with the row-major factor F = L^-1 (Cholesky; made once per tensor with a triangular solve
            // against the identity, setup like the factorisation itself) or F = diag(w)^-1/2 V^T (eigen-decomposed metric):
            // two streaming passes of the hand-written kernels, no library call per J build
            const double* F = d->d_W;
            int nk = d->naux;
            if (d->fac_chol) {
                if (!d->d_Linv) {
                    double* X = (double*)dev_alloc((size_t)nas * nas * 8);
                    dev_zero(X, (size_t)nas * nas * 8, st);
                    IdentityFn idf{X, nas};
                    launch_1d(nas, idf, st);
                    const double one = 1.0;
                    CKB(cublasDtrsm(d->cublas, CUBLAS_SIDE_LEFT, CUBLAS_FILL_MODE_LOWER, CUBLAS_OP_N, CUBLAS_DIAG_NON_UNIT, nas, nas, &one, d->d_fac, nas, X, nas));
                    d->d_Linv = (double*)dev_alloc((size_t)nas * nas * 8);
                    TransposeFn tr{X, d->d_Linv, nas, nas};      // column-major X = row-major X^T: Linv[i][j] = X(i,j)
                    launch_1d((long)nas * nas, tr, st);
                    CK(cudaStreamSynchronize(st));
                    dev_free(X);
                }
                F = d->d_Linv; nk = nas;
            }
            double* d_tmp = (double*)dev_alloc((size_t)std::max(nk, 1) * n_dm * 8);
            dev_zero(d_tmp, (size_t)std::max(nk, 1) * n_dm * 8, st);
            rows_dot(F, nk, nas, d_rho, nas, d_tmp, nk, n_dm, st);
            dev_zero(d_rho, (size_t)nas * n_dm * 8, st);
            cols_acc(F, nk, nas, d_tmp, nk, d_rho, nas, n_dm, st);
            CK(cudaStreamSynchronize(st));
            dev_free(d_tmp);
        }
#else
        for (int s = 0; s < n_dm; s++) {   // L L^T x = b with the row-major lower factor
            double* x = d_rho + (size_t)s * nas;
            const double* L = d->d_fac;
            for (int i = 0; i < nas; i++) { double a = x[i]; for (int k = 0; k < i; k++) a -= L[(size_t)i * nas + k] * x[k]; x[i] = a / L[(size_t)i * nas + i]; }
            for (int i = nas - 1; i >= 0; i--) { double a = x[i]; for (int k = i + 1; k < nas; k++) a -= L[(size_t)k * nas + i] * x[k]; x[i] = a / L[(size_t)i * nas + i]; }
        }
#endif
        // ---- pass 2: Jc[s][col] = sum_P (P|col) rho[s][P]
        double* d_jc = d_dc;   // reuse
#ifndef B200JK_EMULATE
        dev_zero(d_jc, (size_t)d->rowlen * n_dm * 8, st);   // the accumulation kernel adds
#endif
        for_each_j3c_batch(h, d, d->omega, st, [&](int64_t col0, int64_t cols, const double* d_xa, int, int, int) {
#ifndef B200JK_EMULATE
            cols_acc(d_xa, nas, cols, d_rho, nas, d_jc + col0, d->rowlen, n_dm, st);
#else
            for (int s = 0; s < n_dm; s++)
                for (int64_t c = 0; c < cols; c++) {
                    double acc = 0.0;
                    for (int P = 0; P < nas; P++) acc += d_xa[(size_t)P * cols + c] * d_rho[(size_t)s * nas + P];
                    d_jc[(size_t)s * d->rowlen + col0 + c] = acc;
                }
#endif
        });
        dev_zero(d_dcart, nc2 * n_dm * 8, st);
        for (int cb = 0; cb < NPC; cb++) {
            const int np = (int)h->pc[cb].all.size();
            if (!np) continue;
            PairScatterFn g{h->pc[cb].d_all, d->d_ao_off[cb], ncart(h->pc[cb].la), ncart(h->pc[cb].lb), nc, d_jc, d_dcart, d->rowlen, np};
            launch_1d((long)n_dm * np * g.ni * g.nj, g, st);
        }
        Cart2SphFn c2s{d_dcart, d_dsph, ns, nc, 1.0, 0, h->d_sph_sh, h->d_sph_m, h->d_sh_l, h->d_sh_cart, h->d_c2s_off, h->d_c2s};
        launch_1d((long)ns2 * n_dm, c2s, st);
        d2h(vj, d_dsph, ns2 * n_dm * 8, st);
#ifndef B200JK_EMULATE
        CK(cudaStreamSynchronize(st));
#endif
        dev_free(d_dsph); dev_free(d_dcart); dev_free(d_dc); dev_free(d_rho);
        h->stats.ms_total = std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now() - t0).count();
    } catch (std::exception& e) { set_err(h, e.what()); return 2; }
    return 0;
}

extern "C" int b200jk_df_naux(b200jk_handle h, int* naux)
{
    if (!h || !h->df || !naux) { set_err(h, "call b200jk_df_build first"); return 1; }
    *naux = h->df->naux;
    return 0;
}

// A tensor made elsewhere (PySCF's with_df._cderi, an earlier run) handed to the handle instead of b200jk_df_build:
// cderi[naux][nao(nao+1)/2], the reference layout (pyscf/df/incore.py:134-136; assignment test pyscf/df/test/test_df_jk.py:135-142).
// With a shard set, only this rank's rows [naux r/w, naux (r+1)/w) are copied to the device.  No auxiliary basis and no
// metric are attached, so the integral-direct J (b200jk_df_direct_j) is not available on such a handle.
extern "C" int b200jk_df_set_cderi(b200jk_handle h, const double* cderi, int naux, int nao)
{
    if (!h) return 1;
    try {
        if (!cderi || naux < 1) throw std::runtime_error("bad arguments");
        if (nao != h->nsph) throw std::runtime_error("nao does not match the basis of this handle");
        if (h->df) { df_free(h->df); h->df = nullptr; }
        DFState* d = new DFState();
        h->df = d; h->df_free = df_free;
#ifndef B200JK_EMULATE
        CK(cudaSetDevice(h->device));
        cudaStream_t st = h->stream;
        CKB(cublasCreate(&d->cublas));
        CKS(cusolverDnCreate(&d->cusolver));
#else
        stream_t st = 0;
#endif
        d->npair = (long)nao * (nao + 1) / 2;
        d->ncol = d->npair;     // an assigned tensor stays dense: pair screening applies to tensors built here
        d->naux = naux;
        const int bw = h->shard_world, br = h->shard_rank;
        int r_lo, r_hi;
        shard_range(naux, br, bw, r_lo, r_hi);
        d->build_rank = br; d->build_world = bw; d->row0 = r_lo; d->nrow = r_hi - r_lo;
        const std::string split_err = d->rows.plan(h, d->nrow, d->ncol, d->k_slices, false, &d->d_cderi, st);
        if (!split_err.empty()) { df_free(d); h->df = nullptr; throw std::runtime_error(split_err); }
        const int n_dev = d->rows.n_dev;
        if (n_dev > 0) h2d(d->d_cderi, cderi + (size_t)r_lo * d->npair, (size_t)n_dev * d->npair * 8, st);
        if (d->nrow > n_dev)
            memcpy(d->rows.host_row(n_dev), cderi + (size_t)(r_lo + n_dev) * d->npair, (size_t)(d->nrow - n_dev) * d->npair * 8);
#ifndef B200JK_EMULATE
        CK(cudaStreamSynchronize(st));
#endif
    } catch (std::exception& e) { set_err(h, e.what()); return 2; }
    return 0;
}

extern "C" int b200jk_df_local_rows(b200jk_handle h, int* row0, int* nrow)
{
    if (!h || !h->df || !row0 || !nrow) { set_err(h, "call b200jk_df_build first"); return 1; }
    *row0 = h->df->row0; *nrow = h->df->nrow;
    return 0;
}

// Columns cols[ncols] (packed AO-pair indices mu(mu+1)/2+nu) of all LOCAL rows: out[nrow][ncols] — what numpy slicing
// dfobj._cderi[:, cols] gives on the reference's ndarray tensor (pyscf/df/df.py:116); samples a tensor too large to copy.
// Under pair screening a dropped column reads as exact zeros.
struct GatherColsFn {   // cols: positions in the stored rows of length ld, -1 for a column that is not stored (0)
    const double* cderi; const long* cols; double* out; long ld; int ncols;
    B2_HD void operator()(long idx) const
    {
        long r = idx / ncols; int c = (int)(idx - r * ncols);
        out[idx] = cols[c] >= 0 ? cderi[r * ld + cols[c]] : 0.0;
    }
};
extern "C" int b200jk_df_get_cderi_cols(b200jk_handle h, double* out, const int64_t* cols, int ncols)
{
    if (!h || !h->df || !h->df->d_cderi) { set_err(h, "call b200jk_df_build first"); return 1; }
    try {
        DFState* d = h->df;
        if (!out || !cols || ncols < 1) throw std::runtime_error("bad arguments");
        for (int c = 0; c < ncols; c++)
            if (cols[c] < 0 || cols[c] >= d->npair) throw std::runtime_error("column index out of range");
        if (d->nrow < 1) return 0;
        static_assert(sizeof(long) == sizeof(int64_t), "LP64");
        std::vector<long> pos(cols, cols + ncols);     // positions in the stored rows
        if (d->d_col_of)
            for (long& p : pos) p = d->col_of_h[(size_t)p];
        const int n_dev = d->rows.n_dev;
        if (n_dev > 0) {
            long* d_cols = (long*)dev_alloc((size_t)ncols * 8);
            double* d_out = (double*)dev_alloc((size_t)n_dev * ncols * 8);
            h2d(d_cols, pos.data(), (size_t)ncols * 8);
            GatherColsFn g{d->d_cderi, d_cols, d_out, d->ncol, ncols};
            launch_1d((long)n_dev * ncols, g, 0);
            d2h(out, d_out, (size_t)n_dev * ncols * 8);
            dev_sync();
            dev_free(d_cols); dev_free(d_out);
        }
        for (long r = n_dev; r < d->nrow; r++)      // rows in pinned host memory
            for (int c = 0; c < ncols; c++) out[r * ncols + c] = pos[c] >= 0 ? d->rows.host_row(r)[pos[c]] : 0.0;
    } catch (std::exception& e) { set_err(h, e.what()); return 2; }
    return 0;
}

// cderi rows [r0, r0+nr) copied to the host in the reference layout [nr][nao(nao+1)/2] (tests, interchange with PySCF's
// with_df._cderi); a pair-screened tensor is expanded, with exact zeros at the dropped columns
extern "C" int b200jk_df_get_cderi(b200jk_handle h, double* out, int r0, int nr)
{
    if (!h || !h->df || !h->df->d_cderi) { set_err(h, "call b200jk_df_build first"); return 1; }
    try {
        DFState* d = h->df;
        if (r0 < 0 || nr < 0 || r0 + nr > d->nrow) throw std::runtime_error("row range out of bounds (rows are local to this rank)");
        const long ld = d->ncol;
        std::vector<double> packed(d->d_col_of ? (size_t)nr * ld : 0);
        d->rows.read(d->d_col_of ? packed.data() : out, d->d_cderi, r0, nr);   // the stored rows, expanded below when pair-screened
        if (d->d_col_of) {
            memset(out, 0, (size_t)nr * d->npair * 8);
            for (long r = 0; r < nr; r++)
                for (long c = 0; c < ld; c++) out[r * d->npair + d->pk_of_h[(size_t)c]] = packed[(size_t)(r * ld + c)];
        }
    } catch (std::exception& e) { set_err(h, e.what()); return 2; }
    return 0;
}

// ---- J/K from the tensor ------------------------------------------------------------------------
// copies between the J/K workspaces and the caller's arrays, in host memory or, for b200jk_df_jk_device, on the device
static void copy_in(void* dst, const void* src, size_t n, bool on_device, stream_t st) { if (on_device) d2d(dst, src, n, st); else h2d(dst, src, n, st); }
static void copy_out(void* dst, const void* src, size_t n, bool on_device, stream_t st) { if (on_device) d2d(dst, src, n, st); else d2h(dst, src, n, st); }

// one J/K call: its shape and options, shared by the J part and the K engines
struct JKCall {
    DFState* d;
    int nao, n_dm; long n2;
    long ld; const int* col_of;   // stored row length: npair, or the kept columns of a pair-screened tensor (col_of != nullptr)
    int naux;                     // rows held locally (stride of rho)
    int r_lo, kb;                 // first row of this rank's range; rows per K block
    bool use_occ; int nocc, ncol; // K from the orbitals (ncol = nocc) or from the density itself (ncol = nao)
    bool k_sym;                   // K is symmetric: the int8 engine computes its upper triangle, mirrored at the end
    bool tc;                      // the int8-slice engine (k_mode 1), else the FP64 one
    bool on_device;
    stream_t st;
    uint64_t launches;
};

// J, after the rows: unpack J~ and hand it to the caller
static void finish_j(JKCall& c, double* vj)
{
    UnpackTrilFn uf{c.d->d_vjtril, c.d->d_vj, c.nao, c.ld, c.col_of};     // a dropped pair gets J = 0
    launch_1d((long)c.n_dm * c.n2, uf, c.st); c.launches++;
    copy_out(vj, c.d->d_vj, (size_t)c.n_dm * c.n2 * 8, c.on_device, c.st);
}

// J, before the walk: the packed density and zeroed accumulators
static void j_prepare(JKCall& c)
{
    DFState* d = c.d;
    DmTrilFn tf{d->d_dm, d->d_dmtril, c.nao, c.ld, d->d_pk_of};     // pair screening: the kept columns only
    launch_1d((long)c.n_dm * c.ld, tf, c.st); c.launches++;
    dev_zero(d->d_vjtril, (size_t)c.n_dm * c.ld * 8, c.st);
    dev_zero(d->d_rho, (size_t)c.n_dm * c.naux * 8, c.st);
}

#ifndef B200JK_EMULATE
// J of the rows [r0, r0 + nr) at src (row r0 first): rho, then J~ += rho . rows — two streaming passes, both HBM-bound
static void j_rows(JKCall& c, const double* src, int r0, int nr)
{
    DFState* d = c.d;
    d->timer.mark(B200JK_DF_STAGE_J_RHO, c.st);
    rows_dot(src, nr, c.ld, d->d_dmtril, c.ld, d->d_rho + r0, c.naux, c.n_dm, c.st);
    c.launches += (nr + 32768L * DFJ_R - 1) / (32768L * DFJ_R);
    d->timer.mark(B200JK_DF_STAGE_J_ACC, c.st);
    cols_acc(src, nr, c.ld, d->d_rho + r0, c.naux, d->d_vjtril, c.ld, c.n_dm, c.st);
    c.launches++;
    d->timer.mark(-1, c.st);
}

// Keep the int8 slices of as many packed device rows of this rank's range as fit (7 B per unpacked element) resident in SA:
// all of them when the tensor is small or sharded over enough GPUs; otherwise a leading part, the rest being re-cut block by
// block every call.  Decided again when the range, the slice count or the caps of b200jk_df_set_kblock change.
static void resident_slices(JKCall& c, int r_hi)
{
    DFState* d = c.d;
    if (d->sa_decided && d->sa_ns == d->k_slices && d->sa_lo == c.r_lo && d->sa_hi == r_hi) return;
    const int nao = c.nao;
    size_t freeb = 0, totb = 0;
    CK(cudaMemGetInfo(&freeb, &totb));
    freeb += d->SA.cap;                                         // an earlier stack of this handle is reused
    const size_t per_row = slice_row_bytes(nao, d->k_slices);
    const size_t reserve = k_reserve_bytes(nao, c.kb, d->k_slices);   // the per-block stack + workspaces allocated later
    const long nloc = d->rows.dev_end(c.r_lo, r_hi) - c.r_lo;   // only rows in HBM can be resident
    long np = 0;
    if (freeb * 0.85 > (double)reserve) np = (long)((freeb * 0.85 - (double)reserve) / (double)per_row);
    if (np >= nloc) np = nloc;
    else if (np < nloc / 10) np = 0;                            // not worth a second code path
    if (d->np_max >= 0) np = std::min(np, (long)d->np_max);
    while (np > 0 && (size_t)np * nao >= (1UL << 31) - 256) np--;   // row index of the stack is an int
    d->sa_np = (int)np;
    if (np > 0) {
        const size_t kp = ((size_t)nao + 127) / 128 * 128, rows_p = (size_t)np * nao, rp = ((rows_p + 255) / 256) * 256;
        d->SA.alloc((int)rows_p, nao, d->k_slices);
        CK(cudaMemsetAsync(d->SA.q, 0, (size_t)d->k_slices * rp * kp, c.st));
        CK(cudaMemsetAsync(d->SA.E, 0, rp * 4, c.st));
        i8g::split_packed_into(d->SA, 0, d->d_cderi + (size_t)c.r_lo * c.ld, c.ld, nao, (int)np, d->d_rowexp + (size_t)c.r_lo * nao, c.st, c.col_of);
    }
    d->sa_decided = true; d->sa_ns = d->k_slices; d->sa_lo = c.r_lo; d->sa_hi = r_hi;
}

// buffers of the int8 engine: stage 2 in one K range needs pairs(<=ns) * K * 64*64 <= 2^31 - 1 (gemm_ar_acc splits K further
// where this does not hold; gemm_ar rejects a stage 1 whose nao breaks the bound); the slice exponents of the device rows are
// made once (host rows: per staged block, every call)
static void i8_prepare(JKCall& c, int r_hi)
{
    DFState* d = c.d;
    const int nao = c.nao;
    const int kmax = (int)(((1L << 31) - 1) / (4096L * d->k_slices));
    c.kb = std::max(1, std::min(c.kb, kmax / ((c.ncol + 15) & ~15)));   // stage 2 contracts over (P, i) with i padded to 16
    if ((size_t)c.kb * c.ncol * nao > d->y2_cap) { dev_free(d->d_Y2); d->y2_cap = (size_t)c.kb * c.ncol * nao; d->d_Y2 = (double*)dev_alloc(d->y2_cap * 8); }
    if ((size_t)c.ncol * nao > d->occT_cap) { dev_free(d->d_occT); d->occT_cap = (size_t)c.ncol * nao; d->d_occT = (double*)dev_alloc(d->occT_cap * 8); }
    if (!d->d_rowexp) {
        d->d_rowexp = (int*)dev_alloc((size_t)std::max(d->nrow, 1) * nao * 4);
        d->d_rownorm2 = (float*)dev_alloc((size_t)std::max(d->nrow, 1) * nao * 4);
        d->d_cmax2 = (double*)dev_alloc(8);
        if (d->rows.n_dev == d->nrow || d->rows.n_dev > 0)
            i8g::packed_rowexp(d->d_cderi, c.ld, nao, d->rows.n_dev, d->d_rowexp, d->d_rownorm2, c.st, c.col_of);
    }
    resident_slices(c, r_hi);
}

// int8-slice engine on the rows [r0, r0 + nr) at src: the occupied-orbital algorithm when the density carries its orbitals
// (pyscf/df/df_jk.py:339-357), else the general-density algorithm (df_jk.py:382-408) with the density itself as the right
// factor: Y[nu,(P,k)] = sum_mu A_P[nu,mu] D[mu,k], K[i,l] = sum_(P,k) Y[i,(P,k)] A_P[l,k] — the same two int8-slice GEMM
// stages, no cuBLAS
static void k_block_i8(JKCall& c, const double* src, int r0, int nr)
{
    static const bool fuse_y = getenv("B200JK_NO_YFUSE") == nullptr;   // stage 1 cuts the int8 slices of Y itself
    DFState* d = c.d;
    const int nao = c.nao, ncol = c.ncol, ns = d->k_slices;
    const cudaStream_t st = c.st;
    const bool resident = r0 - c.r_lo + nr <= d->sa_np;
    if (!resident) {    // slices of this block straight from the packed rows
        d->timer.mark(B200JK_DF_STAGE_K_SLICE, st);
        i8g::split_packed(d->SAt, src, c.ld, nao, nr, d->d_rowexp + (size_t)r0 * nao, ns, st, c.col_of);
        d->timer.mark(-1, st);
        c.launches++;
    }
    if (!c.use_occ) {   // general density: the block once more as nao long rows G[l][(P,k)] = A_P[l][k]
        d->timer.mark(B200JK_DF_STAGE_K_SLICE, st);
        // same (P, k) column layout as Y: k padded to 16 when stage 1 cuts the slices of Y itself
        const int gcol = fuse_y ? ((nao + 15) & ~15) : nao;
        UnpackLongFn ul{src, d->d_A, nao, c.ld, 0, (long)nr * gcol, gcol, c.col_of};
        launch_1d((long)nao * nr * gcol, ul, st);
        i8g::split_rows(d->SG, d->d_A, (long)nr * gcol, nao, nr * gcol, ns, st);
        d->timer.mark(-1, st);
        c.launches += 2;
    }
    const i8g::SliceStack& A = resident ? d->SA : d->SAt;
    const int a0 = resident ? (r0 - c.r_lo) * nao : 0;
    for (int s = 0; s < c.n_dm; s++) {
        // Y2[nu][(P,i)] = sum_mu A_P[nu,mu] Ct[i,mu] ; K += Y2 Y2^T (upper triangle)
        if (r0 == c.r_lo || c.n_dm > 1) {
            // right factor of stage 1 as rows [ncol][nao]: C~^T, or D^T for the general-density algorithm
            TransposeFn tr{c.use_occ ? d->d_occ + (size_t)s * nao * c.nocc : d->d_dm + (size_t)s * c.n2, d->d_occT, nao, ncol};
            launch_1d((long)nao * ncol, tr, st);
            i8g::split_rows(d->SC, d->d_occT, nao, ncol, nao, ns, st); c.launches += 2;
            i8g::colnorm_max(d->d_occT, nao, ncol, nao, d->d_cmax2, st);
        }
        d->timer.mark(B200JK_DF_STAGE_K_GEMM1, st);
        if (fuse_y) {
            // the row exponents of Y are bounded BEFORE the GEMM (||A_P[nu,:]||_2 max_i ||C~_i||_2), fp64 Y is never written
            const int ncolp = (ncol + 15) & ~15;
            i8g::y_prepare(d->SY, nao, nr, ncolp, ns, d->d_rownorm2 + (size_t)r0 * nao, d->d_cmax2, st);
            i8g::gemm_ar(A, a0, nr * nao, d->SC, nullptr, 0, nao, st, nullptr, &d->SY, ncolp);
            d->timer.mark(B200JK_DF_STAGE_K_SLICE, st);
        } else {
            // stage 1 leaves the row maxima of Y behind (GemmParams::rowmax): the slicing of Y is one pass
            const bool premax = (long)nr * ncol >= 8192;
            if (premax) i8g::split_rows_prepare(d->SY, nao, nr * ncol, ns, st);
            i8g::gemm_ar(A, a0, nr * nao, d->SC, d->d_Y2, (long)nr * ncol, nao, st, premax ? d->SY.maxbits : nullptr);
            d->timer.mark(B200JK_DF_STAGE_K_SLICE, st);
            if (premax) i8g::split_rows_premax(d->SY, d->d_Y2, (long)nr * ncol, nao, nr * ncol, ns, st);
            else i8g::split_rows(d->SY, d->d_Y2, (long)nr * ncol, nao, nr * ncol, ns, st);
        }
        d->timer.mark(B200JK_DF_STAGE_K_GEMM2, st);
        // K += Y Y^T (orbitals) or Y G^T (general density; only its upper triangle when D, hence K, is symmetric)
        i8g::gemm_ar_acc(d->SY, c.use_occ ? d->SY : d->SG, d->d_vk + (size_t)s * c.n2, nao, c.k_sym, st);
        d->timer.mark(-1, st);
        c.launches += 3;
    }
}

// cuBLAS DGEMM engine (k_mode 0, FP64 pipe) on the rows at src: the yardstick the int8 engine is tested and measured against
static void k_block_dgemm(JKCall& c, const double* src, int nr)
{
    DFState* d = c.d;
    const int nao = c.nao, nocc = c.nocc;
    const long n2 = c.n2;
    UnpackFn up{src, d->d_A, nao, c.ld, 0, c.col_of};
    launch_1d((long)nr * n2, up, c.st); c.launches++;
    const double one = 1.0, zero = 0.0;
    for (int s = 0; s < c.n_dm; s++) {
        if (c.use_occ) {
            // Y_P (col-major [nao, nocc]) = A_P * Ctilde ; buffers: occ row-major [nao,nocc] == col-major [nocc,nao]
            CKB(cublasDgemmStridedBatched(d->cublas, CUBLAS_OP_N, CUBLAS_OP_T, nao, nocc, nao, &one, d->d_A, nao, n2,
                                          d->d_occ + (size_t)s * nao * nocc, nocc, 0, &zero, d->d_Y, nao,
                                          (long long)nao * nocc, nr));
            // K += Z Z^T, Z = [nao, nr*nocc]
            CKB(cublasDgemm(d->cublas, CUBLAS_OP_N, CUBLAS_OP_T, nao, nao, nr * nocc, &one, d->d_Y, nao, d->d_Y, nao, &one,
                            d->d_vk + (size_t)s * n2, nao));
        } else {
            // general dm: T_P = A_P * Dbuf (col-major view), K += sum_P T_P * A_P
            CKB(cublasDgemmStridedBatched(d->cublas, CUBLAS_OP_N, CUBLAS_OP_N, nao, nao, nao, &one, d->d_A, nao, n2,
                                          d->d_dm + (size_t)s * n2, nao, 0, &zero, d->d_Y, nao, n2, nr));
            CKB(cublasDgemm(d->cublas, CUBLAS_OP_N, CUBLAS_OP_T, nao, nao, nr * nao, &one, d->d_Y, nao, d->d_A, nao, &one,
                            d->d_vk + (size_t)s * n2, nao));
        }
        c.launches += 2;
    }
}

static void k_block(JKCall& c, const double* src, int r0, int nr)
{
    if (c.tc) k_block_i8(c, src, r0, nr);
    else k_block_dgemm(c, src, nr);
}
#else
static void j_rows(JKCall& c, const double* src, int, int nr)
{
    DFState* d = c.d;
    const long ld = c.ld;
    for (int s = 0; s < c.n_dm; s++)
        for (int r = 0; r < nr; r++) {
            double acc = 0;
            for (long t = 0; t < ld; t++) acc += src[(size_t)r * ld + t] * d->d_dmtril[(size_t)s * ld + t];
            for (long t = 0; t < ld; t++) d->d_vjtril[(size_t)s * ld + t] += acc * src[(size_t)r * ld + t];
        }
}

// C[m][n] = A[m][k] B (B[k][n], or B[n][k] transposed when bt), or C += A B when add: each element summed in k order
static void host_mm(const double* A, const double* B, double* C, int m, int n, int k, bool bt, bool add)
{
    for (int i = 0; i < m; i++)
        for (int l = 0; l < n; l++) {
            double acc = 0;
            for (int j = 0; j < k; j++) acc += A[(size_t)i * k + j] * (bt ? B[(size_t)l * k + j] : B[(size_t)j * n + l]);
            C[(size_t)i * n + l] = add ? C[(size_t)i * n + l] + acc : acc;
        }
}

// the emulation's engine (tests only), per unpacked row A_P: the occupied-orbital algebra of the int8 engine, Y = A_P C~ and
// K += Y Y^T, so that the host-side handling of mo_coeff / mo_occ is exercised on the CPU as well; else K += A_P D A_P (O(N^4))
static void k_block(JKCall& c, const double* src, int, int nr)
{
    DFState* d = c.d;
    const int nao = c.nao, nocc = c.nocc;
    UnpackFn up{src, d->d_A, nao, c.ld, 0, c.col_of};
    launch_1d((long)nr * c.n2, up, c.st); c.launches++;
    std::vector<double> Y((size_t)nao * c.ncol);
    for (int s = 0; s < c.n_dm; s++)
        for (int r = 0; r < nr; r++) {
            const double* A = d->d_A + (size_t)r * c.n2;
            double* K = d->d_vk + (size_t)s * c.n2;
            if (c.use_occ) {
                host_mm(A, d->d_occ + (size_t)s * nao * nocc, Y.data(), nao, nocc, nao, false, false);
                host_mm(Y.data(), Y.data(), K, nao, nao, nocc, true, true);
            } else {
                host_mm(A, d->d_dm + (size_t)s * c.n2, Y.data(), nao, nao, nao, false, false);
                host_mm(Y.data(), A, K, nao, nao, nao, false, true);
            }
        }
}
#endif

// K, before the walk: the workspaces (rows of A padded to 16 columns for the general-density G operand; Y for the FP64 engine
// only), the orbitals, a zeroed K and the int8 engine's own buffers
static void k_prepare(JKCall& c, const double* occ, int r_hi)
{
    DFState* d = c.d;
    const int nao = c.nao;
    if ((size_t)c.kb > d->ws_rows || (size_t)c.ncol > d->ws_nocc || (size_t)c.n_dm > d->ws_occ_ndm) {
        dev_free(d->d_A); dev_free(d->d_Y); dev_free(d->d_occ);
        d->d_A = (double*)dev_alloc((size_t)c.kb * nao * ((nao + 15) & ~15) * 8);
        d->d_Y = (d->k_mode == 1) ? nullptr : (double*)dev_alloc((size_t)c.kb * c.ncol * nao * 8);
        d->d_occ = (double*)dev_alloc((size_t)c.n_dm * nao * c.ncol * 8);
        d->ws_rows = c.kb; d->ws_nocc = c.ncol; d->ws_occ_ndm = c.n_dm;
    }
    if (c.use_occ) copy_in(d->d_occ, occ, (size_t)c.n_dm * nao * c.nocc * 8, c.on_device, c.st);
    dev_zero(d->d_vk, (size_t)c.n_dm * c.n2 * 8, c.st);
#ifndef B200JK_EMULATE
    if (c.tc) i8_prepare(c, r_hi);
#endif
}

// K of the rows [r0, r0 + nr) at src in blocks of kb rows; staged host rows first get their slice exponents
static void k_rows(JKCall& c, const double* src, int r0, int nr)
{
#ifndef B200JK_EMULATE
    DFState* d = c.d;
    if (c.tc && nr > 0 && r0 >= d->rows.n_dev) {
        i8g::packed_rowexp(src, c.ld, c.nao, nr, d->d_rowexp + (size_t)r0 * c.nao, d->d_rownorm2 + (size_t)r0 * c.nao, c.st, c.col_of);
        c.launches++;
    }
#endif
    for (int q = 0; q < nr; q += c.kb) k_block(c, src + (size_t)q * c.ld, r0 + q, std::min(c.kb, nr - q));
}

// multi-GPU: this rank contracts only the local rows [r_lo, r_hi) and returns partial J/K
static void local_range(b200jk_handle h, const DFState* d, int& r_lo, int& r_hi)
{
    if (d->build_world == h->shard_world && d->build_rank == h->shard_rank) { r_lo = 0; r_hi = d->nrow; }
    else if (d->build_world == 1) shard_range(d->nrow, h->shard_rank, h->shard_world, r_lo, r_hi);
    else throw std::runtime_error("the tensor was built for a different shard; call b200jk_df_build again after b200jk_set_shard");
}

static int df_jk_impl(b200jk_handle h, const double* dm, int n_dm, int nao, const double* occ, int nocc, int hermi,
                      double* vj, double* vk, bool on_device)
{
    if (!h) return 1;
    try {
        DFState* d = h->df;
        if (!d || !d->d_cderi) throw std::runtime_error("call b200jk_df_build before b200jk_df_jk");
        if (nao != h->nsph) throw std::runtime_error("nao does not match the basis of this handle");
        if (n_dm < 1) throw std::runtime_error("n_dm < 1");
        auto t0 = std::chrono::steady_clock::now();
        int r_lo, r_hi;
        local_range(h, d, r_lo, r_hi);
#ifndef B200JK_EMULATE
        CK(cudaSetDevice(h->device));
        cudaStream_t st = h->stream;
        CKB(cublasSetStream(d->cublas, st));
        const bool tc = d->k_mode == 1;
#else
        stream_t st = 0;
        const bool tc = false;     // the emulation runs its host engine
#endif
        const bool use_occ = (occ != nullptr && nocc > 0);
        JKCall c{d, nao, n_dm, (long)nao * nao, d->ncol, d->d_col_of, std::max(d->nrow, 1), r_lo, k_block_rows(nao, d->nrow),
                 use_occ, nocc, use_occ ? nocc : nao, use_occ || hermi == 1, tc, on_device, st, 0};
        if (d->kb_max > 0) c.kb = std::min(c.kb, d->kb_max);
        if ((size_t)n_dm > d->ws_ndm) {
            for (double** p : {&d->d_dmtril, &d->d_rho, &d->d_vjtril, &d->d_dm, &d->d_vk, &d->d_vj}) { dev_free(*p); *p = nullptr; }
            d->d_dmtril = (double*)dev_alloc((size_t)n_dm * c.ld * 8);
            d->d_vjtril = (double*)dev_alloc((size_t)n_dm * c.ld * 8);
            d->d_rho = (double*)dev_alloc((size_t)n_dm * c.naux * 8);
            d->d_dm = (double*)dev_alloc((size_t)n_dm * c.n2 * 8);
            d->d_vk = (double*)dev_alloc((size_t)n_dm * c.n2 * 8);
            d->d_vj = (double*)dev_alloc((size_t)n_dm * c.n2 * 8);
            d->ws_ndm = n_dm;
        }
        copy_in(d->d_dm, dm, (size_t)n_dm * c.n2 * 8, on_device, st);
#ifndef B200JK_EMULATE
        CK(cudaEventRecord(h->ev0, st));
        d->timer.start();
#endif
        if (vj) j_prepare(c);
        if (vk) k_prepare(c, occ, r_hi);
        // the rows: J in two passes over all device rows, then K in blocks; host rows block by block.  With every row in HBM, J
        // is finished before K starts.
        const bool resident = d->rows.dev_end(r_lo, r_hi) == r_hi;
        const int hb = d->kb_max > 0 ? std::min(d->rows.stage_rows, d->kb_max) : d->rows.stage_rows;
        d->rows.walk(d->d_cderi, r_lo, r_hi, hb, true, st, [&](const double* src, int r0, int nr) {
            if (vj) j_rows(c, src, r0, nr);
            if (vj && resident) finish_j(c, vj);
            if (vk) k_rows(c, src, r0, nr);
        });
        if (vj && !resident) finish_j(c, vj);
        if (vk) {
            if (c.tc && c.k_sym)
                for (int s = 0; s < n_dm; s++) { MirrorUpperFn mf{d->d_vk + (size_t)s * c.n2, nao}; launch_1d(c.n2, mf, st); c.launches++; }
            copy_out(vk, d->d_vk, (size_t)n_dm * c.n2 * 8, on_device, st);
        }
#ifndef B200JK_EMULATE
        CK(cudaEventRecord(h->ev1, st));
        CK(cudaStreamSynchronize(st));
        float ms = 0;
        CK(cudaEventElapsedTime(&ms, h->ev0, h->ev1));
        h->stats.ms_kernels = ms;
        d->timer.read(d->stage_ms, d->stage_n, B200JK_DF_NSTAGE);
        d->rows.read_times();
#endif
        h->stats.ms_total = std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now() - t0).count();
        h->stats.kernel_launches = c.launches;
    } catch (std::exception& e) { set_err(h, e.what()); return 2; }
    return 0;
}

extern "C" int b200jk_df_jk(b200jk_handle h, const double* dm, int n_dm, int nao, const double* occ, int nocc, int hermi,
                            double* vj, double* vk)
{
    return df_jk_impl(h, dm, n_dm, nao, occ, nocc, hermi, vj, vk, false);
}
// same with dm / occ_coeff / vj / vk resident on the device (multi-GPU all-reduce, HBM-resident benchmark)
extern "C" int b200jk_df_jk_device(b200jk_handle h, const double* dm, int n_dm, int nao, const double* occ, int nocc, int hermi,
                                   double* vj, double* vk)
{
    return df_jk_impl(h, dm, n_dm, nao, occ, nocc, hermi, vj, vk, true);
}

extern "C" int b200jk_df_stage_times(b200jk_handle h, double* ms, int* count, int n)
{
    if (!h || !h->df || !ms || !count) { set_err(h, "call b200jk_df_build first"); return 1; }
    for (int i = 0; i < n; i++) {
        ms[i] = i < B200JK_DF_NSTAGE ? h->df->stage_ms[i] : 0.0;
        count[i] = i < B200JK_DF_NSTAGE ? h->df->stage_n[i] : 0;
    }
    return 0;
}

extern "C" int b200jk_df_set_kblock(b200jk_handle h, int max_block_rows, int max_resident_rows)
{
    if (!h || !h->df) { set_err(h, "call b200jk_df_build first"); return 1; }
    if (max_block_rows == 0 || max_block_rows < -1 || max_resident_rows < -1) { set_err(h, "bad block / resident row cap"); return 1; }
    h->df->kb_max = max_block_rows; h->df->np_max = max_resident_rows;
#ifndef B200JK_EMULATE
    h->df->sa_decided = false;     // the resident stack is re-cut on the next K build
#endif
    return 0;
}

extern "C" int b200jk_df_set_device_rows(b200jk_handle h, int max_rows)
{
    if (!h) return 1;
    if (max_rows < -1) { set_err(h, "bad device row cap"); return 1; }
    h->df_dev_rows = max_rows;
    return 0;
}

extern "C" int b200jk_df_set_pair_tol(b200jk_handle h, double tol)
{
    if (!h) return 1;
    if (std::isnan(tol)) { set_err(h, "bad pair tolerance"); return 1; }
    h->df_pair_tol = tol > 0.0 ? tol : 0.0;
    return 0;
}

extern "C" int b200jk_df_set_raw_test(b200jk_handle h, int on)
{
    if (!h) return 1;
    h->df_raw_test = on != 0;
    return 0;
}

extern "C" int b200jk_df_get_metric_test(b200jk_handle h, double* j2c, int naux)
{
    if (!h || !h->df || !j2c) { set_err(h, "call b200jk_df_build first"); return 1; }
    if (!h->df->raw) { set_err(h, "the metric is kept by raw test builds only (b200jk_df_set_raw_test)"); return 1; }
    if (naux != h->df->naux_sph) { set_err(h, "naux does not match the auxiliary basis of the tensor"); return 1; }
    memcpy(j2c, h->df->raw_j2c.data(), (size_t)naux * naux * 8);
    return 0;
}

extern "C" int b200jk_df_pair_stats(b200jk_handle h, int64_t* ncol, int64_t* npair)
{
    if (!h || !h->df || !ncol || !npair) { set_err(h, "call b200jk_df_build first"); return 1; }
    *ncol = h->df->ncol; *npair = h->df->npair;
    return 0;
}

extern "C" int b200jk_df_row_split(b200jk_handle h, int* n_dev, int* n_host)
{
    if (!h || !h->df || !n_dev || !n_host) { set_err(h, "call b200jk_df_build first"); return 1; }
    *n_dev = h->df->rows.n_dev; *n_host = h->df->nrow - h->df->rows.n_dev;
    return 0;
}

extern "C" int b200jk_df_stream_stats(b200jk_handle h, int64_t* bytes, double* copy_ms, double* exposed_ms)
{
    if (!h || !h->df || !bytes || !copy_ms || !exposed_ms) { set_err(h, "call b200jk_df_build first"); return 1; }
    *bytes = h->df->rows.bytes; *copy_ms = h->df->rows.copy_ms; *exposed_ms = h->df->rows.exposed_ms;
    return 0;
}

extern "C" int b200jk_df_set_kmode(b200jk_handle h, int mode, int nslices)
{
    if (!h || !h->df) { set_err(h, "call b200jk_df_build first"); return 1; }
    if (mode < 0 || mode > 1 || nslices < 1 || nslices > 8) { set_err(h, "bad k mode / slice count"); return 1; }
    if (mode != h->df->k_mode) h->df->ws_rows = 0;     // the FP64 engine has a work buffer of its own: re-size the workspaces
    h->df->k_mode = mode; h->df->k_slices = nslices;
    return 0;
}

#include "df_ao2mo.cuh"
#include "df_mp2.cuh"
#include "df_rpa.cuh"
