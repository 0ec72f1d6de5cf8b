// jk_classes.cuh — instantiation and dispatch of the per-class direct J/K kernels.
// One kernel per angular-momentum class (bra pair class >= ket pair class), 55 classes for s..f.
#pragma once
#include <cstdlib>
#include <stdexcept>
#include "jk_swq.cuh"

namespace b200jk {

// lanes doing useful work when a quartet needs g threads (sub-warp packing or whole warps)
constexpr int lane_eff_permille(int g) { return g <= 32 ? (32 / g) * g * 1000 / 32 : g * 1000 / (((g + 31) / 32) * 32); }

// compile-time tuning knobs (tools/build_variant.sh builds A/B libraries with other values)
#ifndef B2_NVMAX
#define B2_NVMAX 30        // largest register block (doubles) of ERI accumulators per thread
#endif
#ifndef B2_WANT_CTAS
#define B2_WANT_CTAS 2     // CTAs per SM a class launch aims for when it sizes the ket chunks (B200JK_WANT_CTAS overrides at run time)
#endif
#ifndef B2_PBMAX
#define B2_PBMAX 1         // largest primitive batch (QClass::PB) of the block kernels; 1 = one primitive quartet per round
#endif
#ifndef B2_CARVEOUT
#define B2_CARVEOUT -1     // shared-memory share (percent) of the L1/shared array requested for the block kernels; -1: per kernel,
#endif                     // the smallest share that holds the CTAs its register budget allows (block_carveout)

// number of bra-component parts per quartet: register block between 15 and 40 doubles (thread-local
// horizontal recurrences are amortised over the block), then maximise lane use
constexpr int choose_np(int ni, int nj, int nkl)
{
    int nab = ni * nj;
    int best = 0, best_eff = -1;
    for (int np = 1; np <= nj; np++) {
        if (nj % np != 0 || nab / np > B2_NVMAX) continue;
        if (best && nab / np < 15) break;
        if (nkl * np > 512) break;
        int eff = lane_eff_permille(nkl * np);
        if (eff > best_eff + 60) { best = np; best_eff = eff; }   // prefer fewer parts unless clearly better packed
    }
    return best ? best : nj;
}

// primitive quartets per phase round (QClass::PB): double while the (root, direction) tasks of the batch still fit in
// ONE round over the lanes reserved for a quartet and the 2-D integral buffers of a CTA stay below 64 KB
constexpr int choose_pb(int g, int nr, int h_bytes, int nslot)
{
    int gp = g <= 32 ? g : ((g + 31) / 32) * 32;
    int pb = 1;
    while (2 * pb <= B2_PBMAX && 2 * pb * 3 * nr <= gp && 2 * pb * h_bytes * nslot <= 64 * 1024) pb *= 2;
    return pb;
}

// SMs of the current device, queried once per device (the CPU emulation models an H100 SXM: 132)
inline long device_sm_count()
{
#ifndef B200JK_EMULATE
    static int cache[64] = {0};
    int dev = 0;
    if (cudaGetDevice(&dev) != cudaSuccess || dev < 0 || dev >= 64) return 132;
    if (!cache[dev]) {
        int n = 0;
        if (cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess || n <= 0) n = 132;
        cache[dev] = n;
    }
    return cache[dev];
#else
    return 132;
#endif
}

// kets per CTA: at least one batch (`unit` kets in flight per CTA), at most `cap`, and small enough that
// the class fills the SMs several times over
inline int pick_kchunk(int nbra, int nket, int unit, int cap)
{
    static const long want_env = getenv("B200JK_WANT_CTAS") ? atol(getenv("B200JK_WANT_CTAS")) : 0;   // tuning experiment
    long want_ctas = device_sm_count() * (want_env > 0 ? want_env : B2_WANT_CTAS);
    long ny = (want_ctas + nbra - 1) / nbra;
    long kc = (nket + ny - 1) / ny;
    if (kc < unit) kc = unit;
    if (kc > cap) kc = cap;
    return (int)kc;
}

// upper bound of the kets one CTA takes: by default unbounded (the block kernels walk their range in sub-chunks of KCH_MAX, the
// thread-per-quartet kernels keep no list); B200JK_KETS_CAP=1 restores the round-1 cap (one list / 512 kets per CTA)
inline int kets_cap(int round1_cap)
{
    static const bool old_cap = getenv("B200JK_KETS_CAP") && atoi(getenv("B200JK_KETS_CAP")) == 1;
    return old_cap ? round1_cap : (1 << 30);
}

template <int LI, int LJ, int LK, int LL>
struct ClassCfg {
    static constexpr int NP = choose_np(ncart(LI), ncart(LJ), ncart(LK) * ncart(LL));
    using C1 = QClass<LI, LJ, LK, LL, NP>;
    // (ff| bra classes stay at one primitive quartet per round: their batched kernels take the NVVM optimiser tens of minutes)
    static constexpr int PB = (LI + LJ >= 6) ? 1 : choose_pb(C1::G, C1::NR, 3 * C1::NR * C1::HSP * 8, GroupCfg<C1>::NSLOT);
    using C = QClass<LI, LJ, LK, LL, NP, PB>;
    using GC = GroupCfg<C>;
    static constexpr int NT = GC::NT;
    // kets examined per CTA: enough batches per group to amortise the prologue and the J[ij] flush
    static constexpr int KC0 = GC::NSLOT * 8;
    static constexpr int KCHUNK = KC0 > KCH_MAX ? KCH_MAX : (KC0 < 64 ? 64 : KC0);
};

#ifndef B200JK_EMULATE
template <class C, bool SR>
__global__ void __launch_bounds__(TpqCfg<C>::NT) jk_tpq_kernel(const KParams P)
{
    const int bx = blockIdx.x * P.shard_world + P.shard_rank;
    if (bx < P.nbra) tpq_block<C, SR>(P, bx, blockIdx.y, blockIdx.z);
}
template <class C, bool SR>
__global__ void __launch_bounds__(SwqCfg<C>::NT) jk_swq_kernel(const KParams P)
{
    const int bx = blockIdx.x * P.shard_world + P.shard_rank;
    if (bx < P.nbra) swq_block<C, SR>(P, bx, blockIdx.y, blockIdx.z);
}
// Register cap per class: `__launch_bounds__(192, 2)` (<= 168 registers, two resident CTAs per SM) for most block kernels.
// The exemptions below are an untuned carry-over, chosen by A/B timing on an earlier GPU generation and not re-timed on the
// H100; for sm_90a, `-Xptxas -v` reports no spills in any capped kernel, and the exempted classes compile to <= 168
// registers uncapped as well.  The other kernels keep the plain bound (an explicit minBlocks = 1 is NOT equivalent: it
// changes ptxas's scheduling).  B2_MINB = 0 / 2 forces one choice for every class (A/B builds).
#ifndef B2_MINB
#define B2_MINB -1   // -1: per-class table below; 0: never cap; 2: cap every kernel of <= 192 threads
#endif
constexpr bool class_caps_registers(int li, int lj, int lk, int ll)
{
    if (B2_MINB == 0) return false;
    if (B2_MINB > 0) return true;
    if (li == 3 && lj == 1) return false;                                   // (fp| bras: 254 registers, spill when capped
    if (li == 3 && lj == 2 && lk == 1 && ll == 0) return false;            // (fd|ps)
    if (li == 3 && lj == 2 && lk == 3 && ll == 1) return false;            // (fd|fp)
    if (li == 2 && lj == 0 && lk == 1 && ll == 1) return false;            // (ds|pp)
    if (li == 1 && lj == 1 && lk == 1 && ll == 1) return false;            // (pp|pp)
    return true;
}
template <class C, bool SR>
__global__ void __launch_bounds__(GroupCfg<C>::NT) jk_class_kernel(const KParams P)
{
    extern __shared__ __align__(16) unsigned char smraw[];
    BlockSmem<C>& sm = *reinterpret_cast<BlockSmem<C>*>(smraw);
    const int bx = blockIdx.x * P.shard_world + P.shard_rank;
    if (bx < P.nbra) jk_block<C, SR>(P, bx, blockIdx.y, sm);
}
// the same kernel compiled for two resident CTAs per SM (<= 168 registers at 192 threads)
template <class C, bool SR>
__global__ void __launch_bounds__(GroupCfg<C>::NT, 2) jk_class_kernel_2cta(const KParams P)
{
    extern __shared__ __align__(16) unsigned char smraw[];
    BlockSmem<C>& sm = *reinterpret_cast<BlockSmem<C>*>(smraw);
    const int bx = blockIdx.x * P.shard_world + P.shard_rank;
    if (bx < P.nbra) jk_block<C, SR>(P, bx, blockIdx.y, sm);
}
#endif

#ifndef B200JK_EMULATE
typedef cudaStream_t b2_stream_t;
#else
typedef int b2_stream_t;
#endif

#ifndef B200JK_EMULATE
inline void b2_check(cudaError_t e, const char* what)
{
    if (e != cudaSuccess) throw std::runtime_error(std::string(what) + ": " + cudaGetErrorString(e));
}

// Shared-memory carve-out (percent of the SM's L1/shared array) of a block kernel: the smallest one that holds as many CTAs as its
// registers and threads allow, so that the rest of the array stays L1 for what the kernels read through it (Rys table rows,
// primitive pairs, density).  The CUDA driver rounds the percentage up to the next capacity the SM supports.
inline int block_carveout(const void* kern, int nt, size_t smem)
{
    int dev = 0, smem_sm = 0, reserved = 0, ctas = 0;
    b2_check(cudaGetDevice(&dev), "cudaGetDevice");
    b2_check(cudaDeviceGetAttribute(&smem_sm, cudaDevAttrMaxSharedMemoryPerMultiprocessor, dev), "cudaDeviceGetAttribute");
    b2_check(cudaDeviceGetAttribute(&reserved, cudaDevAttrReservedSharedMemoryPerBlock, dev), "cudaDeviceGetAttribute");
    b2_check(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&ctas, kern, nt, 0), "cudaOccupancyMaxActiveBlocksPerMultiprocessor");
    const long per_cta = (long)smem + reserved;
    if (ctas * per_cta > smem_sm) ctas = (int)(smem_sm / per_cta);
    if (ctas < 1) ctas = 1;
    const long pct = (100 * ctas * per_cta + smem_sm - 1) / smem_sm;
    return pct < 100 ? (int)pct : 100;
}

// The entry point a block class launches (only that one is instantiated), configured on first use: dynamic shared memory and
// carve-out.  carveout: the percentage set.
typedef void (*block_kernel_t)(const KParams);
template <class C, bool SR>
block_kernel_t block_kernel(int& carveout)
{
    block_kernel_t kern = nullptr;
    if constexpr (GroupCfg<C>::NT <= 192 && class_caps_registers(C::LI, C::LJ, C::LK, C::LL)) kern = jk_class_kernel_2cta<C, SR>;
    else kern = jk_class_kernel<C, SR>;
    static int carve = -1;
    if (carve < 0) {
        const size_t smem = sizeof(BlockSmem<C>);
        b2_check(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem), "cudaFuncSetAttribute");
        static const int carve_env = getenv("B200JK_CARVEOUT") ? atoi(getenv("B200JK_CARVEOUT")) : -1;   // tuning experiment
        int c = carve_env >= 0 ? carve_env : B2_CARVEOUT;
        if (c < 0) c = block_carveout((const void*)kern, GroupCfg<C>::NT, smem);
        b2_check(cudaFuncSetAttribute(kern, cudaFuncAttributePreferredSharedMemoryCarveout, c), "cudaFuncSetAttribute");
        carve = c;
    }
    carveout = carve;
    return kern;
}

template <class C, bool SR>
void launch_block_kernel(const KParams& P, dim3 grid, int nt, size_t smem, b2_stream_t st)
{
    int carveout = 0;
    block_kernel_t kern = block_kernel<C, SR>(carveout);
    kern<<<grid, nt, smem, st>>>(P);
    cudaError_t e = cudaGetLastError();
    if (e != cudaSuccess) throw std::runtime_error(std::string("jk_class_kernel launch: ") + cudaGetErrorString(e));
}
#endif

template <int LI, int LJ, int LK, int LL>
void launch_one(KParams P, b2_stream_t st)
{
    using Cfg = ClassCfg<LI, LJ, LK, LL>;
    using C = typename Cfg::C;
    if constexpr (TpqCfg<C>::eligible) {
        // low angular momentum: one thread per quartet, registers only (jk_tpq.cuh)
        {
            static const int ps_env = getenv("B200JK_TPQ_PSLICE") ? atoi(getenv("B200JK_TPQ_PSLICE")) : 0;   // tuning experiment
            P.pslice = ps_env > 0 ? ps_env : TpqCfg<C>::PSLICE;
        }
        const int nbx = (P.nbra + P.shard_world - 1) / P.shard_world;   // bra pairs of this rank
        P.kchunk = pick_kchunk(nbx, P.nket, TpqCfg<C>::NT, kets_cap(TpqCfg<C>::KCHUNK));
        int ny = (P.nket + P.kchunk - 1) / P.kchunk;
#ifndef B200JK_EMULATE
        dim3 grid(nbx, ny, (P.bra_nprim_max + P.pslice - 1) / P.pslice);
        if (P.omega < 0.0) jk_tpq_kernel<C, true><<<grid, TpqCfg<C>::NT, 0, st>>>(P);   // erfc operator: two root sets
        else jk_tpq_kernel<C, false><<<grid, TpqCfg<C>::NT, 0, st>>>(P);
        cudaError_t e = cudaGetLastError();
        if (e != cudaSuccess) throw std::runtime_error(std::string("jk_tpq_kernel launch: ") + cudaGetErrorString(e));
#else
        (void)st;
        for (int bx = P.shard_rank; bx < P.nbra; bx += P.shard_world)
            for (int by = 0; by < ny; by++)
                for (int bz = 0; bz * P.pslice < P.bra_nprim_max; bz++) {
                    if (P.omega < 0.0) tpq_block<C, true>(P, bx, by, bz);
                    else tpq_block<C, false>(P, bx, by, bz);
                }
#endif
    } else if constexpr (SwqCfg<C>::eligible) {
        // contracted three-root classes too large for one thread: T lanes per quartet, registers only (jk_swq.cuh)
        using W = SwqCfg<C>;
        P.pslice = W::PSLICE;
        const int nbx = (P.nbra + P.shard_world - 1) / P.shard_world;   // bra pairs of this rank
        P.kchunk = pick_kchunk(nbx, P.nket, W::NSLOT, kets_cap(W::KCHUNK));
        int ny = (P.nket + P.kchunk - 1) / P.kchunk;
#ifndef B200JK_EMULATE
        dim3 grid(nbx, ny, (P.bra_nprim_max + P.pslice - 1) / P.pslice);
        if (P.omega < 0.0) jk_swq_kernel<C, true><<<grid, W::NT, 0, st>>>(P);   // erfc operator: two root sets
        else jk_swq_kernel<C, false><<<grid, W::NT, 0, st>>>(P);
        cudaError_t e = cudaGetLastError();
        if (e != cudaSuccess) throw std::runtime_error(std::string("jk_swq_kernel launch: ") + cudaGetErrorString(e));
#else
        (void)st;
        for (int bx = P.shard_rank; bx < P.nbra; bx += P.shard_world)
            for (int by = 0; by < ny; by++)
                for (int bz = 0; bz * P.pslice < P.bra_nprim_max; bz++) {
                    if (P.omega < 0.0) swq_block<C, true>(P, bx, by, bz);
                    else swq_block<C, false>(P, bx, by, bz);
                }
#endif
    } else {
        const int nbx = (P.nbra + P.shard_world - 1) / P.shard_world;
        P.kchunk = pick_kchunk(nbx, P.nket, Cfg::GC::NSLOT, kets_cap(KCH_MAX));
        int ny = (P.nket + P.kchunk - 1) / P.kchunk;
#ifndef B200JK_EMULATE
        size_t smem = sizeof(BlockSmem<C>);
        dim3 grid(nbx, ny);
        if (P.omega < 0.0) launch_block_kernel<C, true>(P, grid, Cfg::NT, smem, st);   // erfc operator: two root sets per primitive quartet
        else launch_block_kernel<C, false>(P, grid, Cfg::NT, smem, st);
#else
        (void)st;
        BlockSmem<C>* sm = new BlockSmem<C>();
        for (int bx = P.shard_rank; bx < P.nbra; bx += P.shard_world)
            for (int by = 0; by < ny; by++) {
                if (P.omega < 0.0) jk_block<C, true>(P, bx, by, *sm);
                else jk_block<C, false>(P, bx, by, *sm);
            }
        delete sm;
#endif
    }
}

// Launch shape of a class as launch_one launches it (the omega >= 0 entry point), out[B2_LAUNCH_INFO_N]:
//   [0] family: 0 thread-per-quartet, 1 block, 2 sub-warp per quartet     [1] threads per CTA     [2] dynamic shared memory per CTA (bytes)
//   [3] registers per thread     [4] local memory per thread (bytes; > 0 means spills)
//   [5] CTAs per SM by the occupancy API under the carve-out set     [6] carve-out set (percent; -1: none)
//   [7] CTAs per SM that registers and threads alone allow     [8] 1 if launched with bra and ket swapped (use_swapped)
// The CPU emulation fills [0]-[2] and [8] only (-1 elsewhere).
constexpr int B2_LAUNCH_INFO_N = 9;
template <int LI, int LJ, int LK, int LL>
void info_one(int* out)
{
    using Cfg = ClassCfg<LI, LJ, LK, LL>;
    using C = typename Cfg::C;
    for (int i = 0; i < B2_LAUNCH_INFO_N; i++) out[i] = -1;
    const void* kern = nullptr;
    size_t smem = 0;
    if constexpr (TpqCfg<C>::eligible) {
        out[0] = 0; out[1] = TpqCfg<C>::NT;
#ifndef B200JK_EMULATE
        kern = (const void*)jk_tpq_kernel<C, false>;
#endif
    } else if constexpr (SwqCfg<C>::eligible) {
        out[0] = 2; out[1] = SwqCfg<C>::NT;
#ifndef B200JK_EMULATE
        kern = (const void*)jk_swq_kernel<C, false>;
#endif
    } else {
        out[0] = 1; out[1] = Cfg::NT; smem = sizeof(BlockSmem<C>);
#ifndef B200JK_EMULATE
        kern = (const void*)block_kernel<C, false>(out[6]);
#endif
    }
    out[2] = (int)smem;
#ifndef B200JK_EMULATE
    cudaFuncAttributes fa;
    b2_check(cudaFuncGetAttributes(&fa, kern), "cudaFuncGetAttributes");
    out[3] = fa.numRegs;
    out[4] = (int)fa.localSizeBytes;
    b2_check(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&out[5], kern, out[1], smem), "cudaOccupancyMaxActiveBlocksPerMultiprocessor");
    b2_check(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&out[7], kern, out[1], 0), "cudaOccupancyMaxActiveBlocksPerMultiprocessor");
#else
    (void)kern;
#endif
}

// pair class id = l1*(l1+1)/2 + l2  (l1 >= l2)
#define B2_PAIR_CASES(X) \
    X(0, 0, 0) X(1, 1, 0) X(2, 1, 1) X(3, 2, 0) X(4, 2, 1) X(5, 2, 2) X(6, 3, 0) X(7, 3, 1) X(8, 3, 2) X(9, 3, 3)

// host-side mirror of TpqCfg<C>::eligible for the class (la lb|lc ld) as launched
inline bool tpq_class(int la, int lb, int lc, int ld)
{
    int nout = ncart(la) * ncart(lb) * ncart(lc) * ncart(ld);
    int nr = (la + lb + lc + ld) / 2 + 1;
    return nout <= 36 && nr <= 3 && choose_np(ncart(la), ncart(lb), ncart(lc) * ncart(ld)) == 1;
}

// Orientation of a class pair (hi id > lo id): by default the larger class is the register-resident bra.  For these
// pairs the opposite choice packs the warps better (threads = fs/fp components instead of dp/dd: 30 of 32 lanes
// instead of 18) and needs fewer reductions per integral, so they run with bra = lo class, ket = hi class.
constexpr bool use_swapped(int hi, int lo)
{
    return (hi == 6 && lo == 4) || (hi == 7 && lo == 4) || (hi == 6 && lo == 2) || (hi == 7 && lo == 5);
}

template <int LI, int LJ>
void launch_ket(int ck, const KParams& P, b2_stream_t st)
{
    constexpr int cb = LI * (LI + 1) / 2 + LJ;
    switch (ck) {
#define X(id, lk, ll)                                                      \
    case id:                                                               \
        if constexpr (id <= cb || use_swapped(id, cb)) launch_one<LI, LJ, lk, ll>(P, st); \
        return;
        B2_PAIR_CASES(X)
#undef X
    }
    throw std::runtime_error("bad ket class");
}

template <int LI, int LJ>
void info_ket(int ck, int* out)
{
    constexpr int cb = LI * (LI + 1) / 2 + LJ;
    switch (ck) {
#define X(id, lk, ll)                                                      \
    case id:                                                               \
        if constexpr (id <= cb || use_swapped(id, cb)) info_one<LI, LJ, lk, ll>(out); \
        return;
        B2_PAIR_CASES(X)
#undef X
    }
    throw std::runtime_error("bad ket class");
}

// one translation unit per bra pair class (jk_class_tu.cu compiled with -DB2_BRA_ID=<id>)
#define X(id, li, lj) void launch_bra_##id(int ck, const KParams& P, b2_stream_t st); void info_bra_##id(int ck, int* out);
B2_PAIR_CASES(X)
#undef X

// launch shape of the class (cb ck), cb >= ck, as launch_class launches it (see info_one)
inline void class_info(int cb, int ck, int* out)
{
    const bool swapped = cb > ck && use_swapped(cb, ck);
    if (swapped) { int t = cb; cb = ck; ck = t; }
    switch (cb) {
#define X(id, li, lj)                  \
    case id:                           \
        info_bra_##id(ck, out);        \
        out[8] = swapped ? 1 : 0;      \
        return;
        B2_PAIR_CASES(X)
#undef X
    }
    throw std::runtime_error("bad bra class");
}

inline void launch_class(int cb, int ck, const KParams& P0, b2_stream_t st)
{
    KParams P = P0;
    if (cb > ck && use_swapped(cb, ck)) {   // run the pair with the smaller class as the stationary bra
        P.bra_pairs = P0.ket_pairs; P.nbra = P0.nket;
        P.ket_pairs = P0.bra_pairs; P.nket = P0.nbra;
        P.bra_nprim_max = P0.ket_nprim_max; P.ket_nprim_max = P0.bra_nprim_max;
        int t = cb; cb = ck; ck = t;
    }
    switch (cb) {
#define X(id, li, lj)                  \
    case id:                           \
        launch_bra_##id(ck, P, st);    \
        return;
        B2_PAIR_CASES(X)
#undef X
    }
    throw std::runtime_error("bad bra class");
}

}  // namespace b200jk
