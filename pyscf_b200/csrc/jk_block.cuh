// jk_block.cuh — the CTA-level procedure of the direct J/K kernels (one template per class).
//
// A CTA owns ONE bra shell pair and a chunk of the ket-pair list, which it screens on device and
// compacts into shared memory.  Inside the CTA, independent thread GROUPS (a sub-warp, one warp, or a
// few warps joined by a named barrier) pull batches of ket pairs from a shared counter; a group only
// ever synchronises with itself, so there is no block-wide lock-step over primitive loops.
// J[ij] for the stationary bra pair is accumulated in registers across all kets and flushed once.
//
// Compiles as a CUDA kernel body and, with B200JK_EMULATE, as a sequential SIMT emulation on the CPU
// (tests only): groups run one after the other and every phase is a loop over the group's lanes.
#pragma once
#include "jk_core.cuh"

namespace b200jk {

constexpr int KCH_MAX = 512;  // ket pairs examined per CTA
#ifndef B2_CTA_THREADS
#define B2_CTA_THREADS 192   // target CTA size of the block kernels (tuning knob)
#endif
#ifndef B2_SMEM_CAP
#define B2_SMEM_CAP 0        // if > 0: fewer groups per CTA so that the quartet slots of a CTA stay below this many bytes
#endif                       // (several small CTAs per SM instead of one that owns all of its shared memory)

struct KParams {
    const ShellPair* bra_pairs; int nbra;
    const ShellPair* ket_pairs; int nket;
    int same_class;
    const PrimPair* prims;
    RysTables tb;
    double omega, tol;
    const double* dmc; int nsh;
    const double* dmj; const double* dmk;
    double* vj; double* vk;
    int n, n_dm_j, n_dm_k;
    int kchunk;
    int bra_nprim_max, ket_nprim_max;
    int shard_rank, shard_world;   // multi-GPU: this rank owns bra pairs bx = i*world + rank (lists are cost-sorted)
    int pslice;                    // thread-per-quartet kernels: bra primitive pairs per CTA slice (blockIdx.z)
    unsigned long long* counters;  // [0] quartets computed, [1] quartets screened out (may be null)
};

constexpr int pow2ceil(int x) { int p = 1; while (p < x) p *= 2; return p; }

#ifndef B2_PPW
#define B2_PPW 0             // 1: "part per warp" lane layout for classes whose bra block is split into NP > 1 parts
#endif

// Lane layout of one thread group.
//  * default: a quartet owns G = NKL * NP consecutive lanes (part index slowest); QPG = 32 / G quartets share a warp when
//    G <= 32, otherwise the quartet gets whole warps.  Lanes of different PARTS then sit in one warp, and since every part
//    is different straight-line code (compile-time Cartesian indices of its j components) the warp runs the root sum
//    once per part it holds (ncu: 20 of 32 threads active per instruction in (fd|dp)).
//  * PPW (B2_PPW, classes with NP > 1 and NKL <= 32): a group is NP warps, warp w holds part w of QPG = 32 / NKL quartets,
//    so no warp ever mixes parts.  Logical lane id inside a quartet stays g = part * NKL + (c,d).
// classes given the part-per-warp layout: chosen by A/B timing of benzene/cc-pVTZ on an earlier GPU generation, not re-measured
// on the H100 (tools/build_variant.sh + tools/ab_direct.py repeat that A/B).
// B2_PPW = 1 forces the layout for every class with NP > 1 (A/B builds), -1 switches it off everywhere.
constexpr bool class_prefers_ppw(int li, int lj, int lk, int ll)
{
    return (li == 2 && lj == 2 && lk == 1 && ll == 1) || (li == 3 && lj == 3 && lk == 2 && ll == 0) || (li == 3 && lj == 2 && lk == 2 && ll == 0) ||
           (li == 2 && lj == 2 && lk == 2 && ll == 1) || (li == 2 && lj == 2 && lk == 2 && ll == 0) || (li == 3 && lj == 2 && lk == 1 && ll == 1);
}
// Classes whose phase E stays one reduction per lane and sum (phase_digest_lane) instead of one per distinct element through
// the slot's scratch (DigestCfg): the five where the scratch rounds, each behind two barriers of a multi-warp group, cost more
// than the reductions they save.  Class times on one H100 80GB HBM3 at 700 W, benzene/cc-pVTZ, classes serialised, best of 3,
// per-lane -> per-element (ms): (fd|dd) 0.763 -> 0.848, (fs|dd) 0.601 -> 0.647, (dd|dp) 1.317 -> 1.355, (fd|fd) 0.463 -> 0.484,
// (dd|dd) 0.390 -> 0.406; the old library's own runs differ by up to 0.02 ms.
constexpr bool class_reduces_per_lane(int li, int lj, int lk, int ll)
{
    return (li == 3 && lj == 2 && lk == 2 && ll == 2) || (li == 3 && lj == 0 && lk == 2 && ll == 2) || (li == 2 && lj == 2 && lk == 2 && ll == 1) ||
           (li == 3 && lj == 2 && lk == 3 && ll == 2) || (li == 2 && lj == 2 && lk == 2 && ll == 2);
}
template <class C>
struct GroupCfg {
    static constexpr int G = C::G;
    static constexpr bool PPW = (B2_PPW > 0 || (B2_PPW == 0 && class_prefers_ppw(C::LI, C::LJ, C::LK, C::LL))) && C::NP > 1 && C::NKL <= 32 && C::NP <= 8;
    static constexpr int GP = G <= 32 ? G : ((G + 31) / 32) * 32;              // lanes reserved per quartet (default layout)
    static constexpr int GW = PPW ? C::NP : (GP + 31) / 32;                  // warps per group
    static constexpr int TG = GW * 32;                                       // threads per group
    static constexpr int QPG = PPW ? 32 / C::NKL : (GP <= 32 ? 32 / GP : 1); // quartets in flight per group
    static constexpr int NG0 = B2_CTA_THREADS / TG;
    static constexpr int NG1 = NG0 < 1 ? 1 : (NG0 > 8 ? 8 : NG0);
    static constexpr int NG2 = (NG1 * QPG > 64) ? ((64 / QPG) < 1 ? 1 : 64 / QPG) : NG1;  // groups per CTA, <= 64 quartet slots
    static constexpr int NGC = B2_SMEM_CAP > 0 ? (int)(B2_SMEM_CAP / (QPG * sizeof(SlotSmem<C>))) : NG2;
    static constexpr int NG = NGC < 1 ? 1 : (NGC < NG2 ? NGC : NG2);
    static constexpr int NT = NG * TG;
    static constexpr int NSLOT = NG * QPG;
    // PPW layout: lane lt of a group -> (quartet sub-slot sl, logical lane g inside the quartet); false for idle lanes
    static B2_HD bool decode(int lt, int& sl, int& g)
    {
        const int w = lt / 32, l = lt % 32;
        sl = l / C::NKL;
        g = w * C::NKL + l % C::NKL;
        if (sl >= QPG) { sl = 0; g = 0; return false; }
        return true;
    }
};

template <class C>
struct BlockSmem {
    SlotSmem<C> slot[GroupCfg<C>::NSLOT];
    BraInfo bra;
    PrimPair bprim[MAX_PRIM_PER_PAIR];                 // the stationary bra pair's primitive pairs (bulk async copy)
    unsigned long long mbar_bra;                        // mbarrier of that copy
    int klist[KCH_MAX];
    int nk;
    int next;
    int gbase[GroupCfg<C>::NG];
};

template <class C>
struct LaneCtx {
    ThreadCtx<C> t;
    double jij[C::NV];
    double jkl;      // phase E: this lane's J[kl] sum of the current density (digest_j)
    int grp, lt, slot, valid;
    int ibp, ikp;
    int sr;          // omega < 0 only: 0 = Coulomb pass, 1 = (negated) erf pass of the current primitive quartet
};

#if defined(__CUDA_ARCH__)
#define B2_ALL_THREADS(tid) { const int tid = threadIdx.x;
#define B2_END }
#define B2_SYNC() __syncthreads()
#define B2_GROUP_LANES(lt) { const int lt = threadIdx.x % GroupCfg<C>::TG;
#define B2_CTX(tid) ctx
template <class C>
__device__ __forceinline__ void group_sync(int grp)
{
    if constexpr (GroupCfg<C>::GW == 1) __syncwarp();
    else asm volatile("bar.sync %0, %1;" ::"r"(grp + 1), "n"(GroupCfg<C>::TG) : "memory");
}
#else
#define B2_ALL_THREADS(tid) for (int tid = 0; tid < GroupCfg<C>::NT; tid++) {
#define B2_END }
#define B2_SYNC()
#define B2_GROUP_LANES(lt) for (int lt = 0; lt < GroupCfg<C>::TG; lt++) {
#define B2_CTX(tid) ctxs[tid]
template <class C>
inline void group_sync(int) {}
#endif

#if defined(__CUDA_ARCH__)
// 1-D bulk asynchronous copy global -> shared (TMA engine, SASS UBLKCP) completing on an mbarrier
__device__ __forceinline__ void bulk_g2s(void* dst, const void* src, unsigned bytes, unsigned long long* bar)
{
    unsigned d = (unsigned)__cvta_generic_to_shared(dst), b = (unsigned)__cvta_generic_to_shared(bar);
    asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(b), "r"(bytes) : "memory");
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
                 ::"r"(d), "l"(src), "r"(bytes), "r"(b) : "memory");
}
__device__ __forceinline__ void bulk_wait(unsigned long long* bar, unsigned parity)
{
    unsigned b = (unsigned)__cvta_generic_to_shared(bar), ok;
    do {
        asm volatile("{\n\t.reg .pred p;\n\tmbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\tselp.u32 %0, 1, 0, p;\n\t}\n"
                     : "=r"(ok) : "r"(b), "r"(parity) : "memory");
    } while (!ok);
}
#endif

// One group's life: pull ket batches until the CTA's list is exhausted.
template <class C, bool SR>
#ifdef __CUDACC__
__device__ __forceinline__
#else
inline
#endif
void group_proc(const KParams& P, BlockSmem<C>& sm, int grp, int nk, int bx,
#if defined(__CUDA_ARCH__)
                LaneCtx<C>& ctx
#else
                LaneCtx<C>* ctxs
#endif
)
{
    using GC = GroupCfg<C>;
    const int nbp = sm.bra.nprim;
    const int tid0 = grp * GC::TG;
    (void)tid0;
    for (;;) {
        B2_GROUP_LANES(lt)
            if (lt == 0) {
#if defined(__CUDA_ARCH__)
                sm.gbase[grp] = atomicAdd(&sm.next, GC::QPG);
#else
                sm.gbase[grp] = sm.next; sm.next += GC::QPG;
#endif
            }
        B2_END
        group_sync<C>(grp);
        const int base = sm.gbase[grp];
        if (base >= nk) break;
        // ---- slot setup
        B2_GROUP_LANES(lt)
            LaneCtx<C>& L = B2_CTX(tid0 + lt);
            if (L.valid) {
                SlotSmem<C>& s = sm.slot[L.slot];
                if (L.t.g == 0) {
                    int e = base + (L.slot - grp * GC::QPG);
                    s.active = (e < nk);
                    if (s.active) {
                        int kk = sm.klist[e];
                        const ShellPair& kp = P.ket_pairs[kk];
                        s.kl = kk; s.k0 = kp.i0; s.l0 = kp.j0;
                        s.nprim_k = kp.nprim; s.prim_off_k = kp.prim_off;
                        s.nq = nbp * kp.nprim * (SR ? 2 : 1);
                        double f = 1.0;
                        if (sm.bra.same) f *= 0.5;
                        if (kp.same) f *= 0.5;
                        if (P.same_class && kk == bx) f *= 0.5;
                        s.fac = f;
                        slot_set_cd<C>(s, kp.ABx, kp.ABy, kp.ABz);
                    } else {
                        s.nprim_k = 0; s.nq = 0;
                    }
                }
                B2_UNROLL
                for (int e = 0; e < C::NV; e++) L.t.v[e] = 0.0;
                L.ibp = 0; L.ikp = 0; L.sr = 0;
            }
        B2_END
        group_sync<C>(grp);
        constexpr bool sr_op = SR;   // erfc = Coulomb - erf: every primitive quartet is visited twice (omega < 0)
        if constexpr (C::PB > 1) {
            // ---- primitive batching: PB primitive quartets per round.  Quartet e of the slot (e < nq) is
            //      (bra primitive ibp, ket primitive ikp, pass sr) with e = (ibp * nprim_k + ikp) * passes + sr,
            //      the same order as the one-at-a-time loop below, so the sums are bit-identical.
            int nqmax = 0;
            for (int q = 0; q < GC::QPG; q++) {
                int n_ = sm.slot[grp * GC::QPG + q].nq;
                nqmax = n_ > nqmax ? n_ : nqmax;
            }
            for (int e0 = 0; e0 < nqmax; e0 += C::PB) {
                // phase A: PB*NR root tasks over the G lanes of each quartet
                B2_GROUP_LANES(lt)
                    LaneCtx<C>& L = B2_CTX(tid0 + lt);
                    if (L.valid) {
                        SlotSmem<C>& s = sm.slot[L.slot];
                        const int nq = s.nq, nkp = s.nprim_k;
                        B2_NOUNROLL
                        for (int task = L.t.g; task < C::PB * C::NR; task += C::G) {
                            const int b = task / C::NR, r = task - b * C::NR;
                            const int e = e0 + b;
                            if (e < nq) {
                                const int sr = sr_op ? (e & 1) : 0;
                                const int pq = sr_op ? (e >> 1) : e;
                                const int ibp = pq / nkp, ikp = pq - ibp * nkp;
                                phase_root_one<C>(s, b, r, sm.bprim[ibp], load_prim(P.prims + s.prim_off_k + ikp), P.tb,
                                                  sr_op ? (sr ? -P.omega : 0.0) : P.omega, (sr_op && sr) ? -1.0 : 1.0);
                            }
                        }
                    }
                B2_END
                group_sync<C>(grp);
                // phase B: PB*3*NR (quartet, root, direction) recurrence tasks
                B2_GROUP_LANES(lt)
                    LaneCtx<C>& L = B2_CTX(tid0 + lt);
                    if (L.valid) {
                        SlotSmem<C>& s = sm.slot[L.slot];
                        const int nq = s.nq;
                        B2_NOUNROLL
                        for (int task = L.t.g; task < C::PB * 3 * C::NR; task += C::G) {
                            const int b = task / (3 * C::NR), rem = task - b * (3 * C::NR);
                            const int r = rem / 3, x = rem - 3 * r;
                            if (e0 + b < nq) vrr_one<C>(s, b, r, x);
                        }
                    }
                B2_END
                group_sync<C>(grp);
                // phase D: every lane sums the batch into its register block
                B2_GROUP_LANES(lt)
                    LaneCtx<C>& L = B2_CTX(tid0 + lt);
                    if (L.valid) {
                        SlotSmem<C>& s = sm.slot[L.slot];
                        const int nq = s.nq;
                        B2_NOUNROLL
                        for (int b = 0; b < C::PB; b++)
                            if (e0 + b < nq) phase_accumulate<C>(s, L.t, sm.bra.ABx, sm.bra.ABy, sm.bra.ABz, b);
                    }
                B2_END
                // the next round's phase A rewrites U/W/pc, which phase B of this round (already behind a barrier) read;
                // H is rewritten only after the barrier that follows phase A
            }
        } else {
        int npmax = 0;
        for (int q = 0; q < GC::QPG; q++) {
            int nk_ = sm.slot[grp * GC::QPG + q].nprim_k;
            npmax = nk_ > npmax ? nk_ : npmax;
        }
        npmax *= nbp;
        if (sr_op) npmax *= 2;

        for (int ip = 0; ip < npmax; ip++) {
            // ---- phase A: Rys roots
            B2_GROUP_LANES(lt)
                LaneCtx<C>& L = B2_CTX(tid0 + lt);
                if (L.valid) {
                    SlotSmem<C>& s = sm.slot[L.slot];
                    if (s.active && L.ibp < nbp)
                        phase_roots<C>(s, L.t.g, sm.bprim[L.ibp], load_prim(P.prims + s.prim_off_k + L.ikp), P.tb,
                                       sr_op ? (L.sr ? -P.omega : 0.0) : P.omega, (sr_op && L.sr) ? -1.0 : 1.0);
                }
            B2_END
            group_sync<C>(grp);
            // ---- phase B: vertical recurrences into shared memory
            B2_GROUP_LANES(lt)
                LaneCtx<C>& L = B2_CTX(tid0 + lt);
                if (L.valid) {
                    SlotSmem<C>& s = sm.slot[L.slot];
                    if (s.active && L.ibp < nbp) phase_vrr<C>(s, L.t.g);
                }
            B2_END
            group_sync<C>(grp);
            // ---- phase D: horizontal recurrences + root sum in registers
            B2_GROUP_LANES(lt)
                LaneCtx<C>& L = B2_CTX(tid0 + lt);
                if (L.valid) {
                    SlotSmem<C>& s = sm.slot[L.slot];
                    if (s.active && L.ibp < nbp) {
                        phase_accumulate<C>(s, L.t, sm.bra.ABx, sm.bra.ABy, sm.bra.ABz);
                        if (sr_op && !L.sr) L.sr = 1;
                        else { L.sr = 0; if (++L.ikp == s.nprim_k) { L.ikp = 0; L.ibp++; } }
                    }
                }
            B2_END
        }
        }
        // ---- phase E: digestion
        if constexpr (class_reduces_per_lane(C::LI, C::LJ, C::LK, C::LL)) {
            B2_GROUP_LANES(lt)
                LaneCtx<C>& L = B2_CTX(tid0 + lt);
                if (L.valid) {
                    SlotSmem<C>& s = sm.slot[L.slot];
                    if (s.active) {
                        if (P.vj) phase_digest_lane<C>(s, L.t, sm.bra.i0, sm.bra.j0, P.n, P.n_dm_j, P.dmj, nullptr, P.vj, nullptr,
                                                       P.n_dm_j == 1 ? L.jij : nullptr);
                        if (P.vk) phase_digest_lane<C>(s, L.t, sm.bra.i0, sm.bra.j0, P.n, P.n_dm_k, nullptr, P.dmk, nullptr, P.vk, nullptr);
                    }
                }
            B2_END
        } else {
            // one density at a time: the lanes' sums go through the slot's scratch in NRND rounds, and one lane per distinct
            // K / J[kl] element issues its reduction (DigestCfg)
            using DG = DigestCfg<C>;
            const int ndm_j = P.vj ? P.n_dm_j : 0, ndm_k = P.vk ? P.n_dm_k : 0;
            const size_t n2 = (size_t)P.n * P.n;
            for (int idm = 0; idm < (ndm_j > ndm_k ? ndm_j : ndm_k); idm++) {
                const double* Dj = idm < ndm_j ? P.dmj + idm * n2 : nullptr;
                const double* Dk = idm < ndm_k ? P.dmk + idm * n2 : nullptr;
                double* J = idm < ndm_j ? P.vj + idm * n2 : nullptr;
                double* K = idm < ndm_k ? P.vk + idm * n2 : nullptr;
                B2_GROUP_LANES(lt)
                    LaneCtx<C>& L = B2_CTX(tid0 + lt);
                    L.jkl = 0.0;
                    if (L.valid && Dj) {
                        const SlotSmem<C>& s = sm.slot[L.slot];
                        if (s.active) L.jkl = digest_j<C>(s, L.t, sm.bra.i0, sm.bra.j0, P.n, Dj, J, P.n_dm_j == 1 ? L.jij : nullptr);
                    }
                B2_END
                B2_UNROLL
                for (int rnd = 0; rnd < DG::NRND; rnd++) {
                    group_sync<C>(grp);   // phase D, or the previous round's flush, is done with H
                    B2_GROUP_LANES(lt)
                        LaneCtx<C>& L = B2_CTX(tid0 + lt);
                        if (L.valid) {
                            SlotSmem<C>& s = sm.slot[L.slot];
                            if (s.active) phase_digest<C>(s, L.t, rnd * DG::RPR, sm.bra.i0, sm.bra.j0, P.n, Dk, L.jkl);
                        }
                    B2_END
                    group_sync<C>(grp);
                    B2_GROUP_LANES(lt)
                        LaneCtx<C>& L = B2_CTX(tid0 + lt);
                        if (L.valid) {
                            const SlotSmem<C>& s = sm.slot[L.slot];
                            if (s.active) digest_flush<C>(s, L.t.g, rnd * DG::RPR, sm.bra.i0, sm.bra.j0, P.n, J, K);
                        }
                    B2_END
                }
            }
        }
        group_sync<C>(grp);
    }
}

template <class C, bool SR>
#ifdef __CUDACC__
__device__ __forceinline__
#else
inline
#endif
void jk_block(const KParams& P, int bx, int by, BlockSmem<C>& sm)
{
    using GC = GroupCfg<C>;
    const ShellPair& bpair = P.bra_pairs[bx];
    const int kmax = P.same_class ? (bx + 1) : P.nket;
    const int kbeg = by * P.kchunk;
    const int kend = (kbeg + P.kchunk < kmax) ? kbeg + P.kchunk : kmax;
    if (kbeg >= kend) return;
#if defined(__CUDA_ARCH__)
    LaneCtx<C> ctx;
#else
    LaneCtx<C>* ctxs = new LaneCtx<C>[GC::NT];
#endif

    B2_ALL_THREADS(tid)
        LaneCtx<C>& L = B2_CTX(tid);
        L.grp = tid / GC::TG;
        L.lt = tid % GC::TG;
        if constexpr (GC::PPW) {
            int sl, g;
            L.valid = GC::decode(L.lt, sl, g);
            L.slot = L.grp * GC::QPG + sl;
            thread_decode<C>(L.t, g);
        } else {
            int sl = L.lt / GC::GP, g = L.lt % GC::GP;
            L.valid = (sl < GC::QPG) && (g < C::G);
            L.slot = L.grp * GC::QPG + (sl < GC::QPG ? sl : 0);
            thread_decode<C>(L.t, g < C::G ? g : 0);
        }
        L.t.q = L.slot;
        B2_UNROLL
        for (int e = 0; e < C::NV; e++) L.jij[e] = 0.0;
        if (tid == 0) {
            sm.bra.ABx = bpair.ABx; sm.bra.ABy = bpair.ABy; sm.bra.ABz = bpair.ABz;
            sm.bra.i0 = bpair.i0; sm.bra.j0 = bpair.j0;
            sm.bra.nprim = bpair.nprim; sm.bra.prim_off = bpair.prim_off;
            sm.bra.same = bpair.same; sm.bra.idx = bx;
            sm.nk = 0; sm.next = 0;
#if defined(__CUDA_ARCH__)
            {
                unsigned a = (unsigned)__cvta_generic_to_shared(&sm.mbar_bra);
                asm volatile("mbarrier.init.shared::cta.b64 [%0], 1;" ::"r"(a));
            }
            asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
            bulk_g2s(sm.bprim, P.prims + bpair.prim_off, (unsigned)bpair.nprim * (unsigned)sizeof(PrimPair), &sm.mbar_bra);
#else
            for (int e2 = 0; e2 < bpair.nprim; e2++) sm.bprim[e2] = P.prims[bpair.prim_off + e2];
#endif
        }
    B2_END
    B2_SYNC();
#if defined(__CUDA_ARCH__)
    bulk_wait(&sm.mbar_bra, 0);
#endif

    // The CTA's ket range may be longer than the shared list: it is walked in sub-chunks of KCH_MAX kets (screen, compact,
    // process), the stationary J[ij] block staying in registers across all of them.  Fewer, longer CTAs amortise the per-CTA
    // prologue and the drain of the last batches.
    for (int sub = kbeg; sub < kend; sub += KCH_MAX) {
        const int send = (sub + KCH_MAX < kend) ? sub + KCH_MAX : kend;
        if (sub > kbeg) {
            B2_SYNC();      // every group has left group_proc: the list and the batch counter can be reset
            B2_ALL_THREADS(tid)
                if (tid == 0) { sm.nk = 0; sm.next = 0; }
            B2_END
            B2_SYNC();
        }
        // ---- on-device screening: compact the surviving kets of this sub-chunk
        B2_ALL_THREADS(tid)
            for (int kk = sub + tid; kk < send; kk += GC::NT) {
                const ShellPair& kp = P.ket_pairs[kk];
                bool keep = keep_quartet(bpair.q, kp.q, bpair.ish, bpair.jsh, kp.ish, kp.jsh, P.dmc, P.nsh, P.tol,
                                         P.vj != nullptr, P.vk != nullptr);
                if (keep) {
#if defined(__CUDA_ARCH__)
                    int pos = atomicAdd(&sm.nk, 1);
#else
                    int pos = sm.nk++;
#endif
                    sm.klist[pos] = kk;
                }
            }
        B2_END
        B2_SYNC();
        const int nk = sm.nk;
#if defined(__CUDA_ARCH__)
        if (P.counters && threadIdx.x == 0) {
            atomicAdd(&P.counters[0], (unsigned long long)nk);
            atomicAdd(&P.counters[1], (unsigned long long)(send - sub - nk));
        }
        group_proc<C, SR>(P, sm, threadIdx.x / GC::TG, nk, bx, ctx);
#else
        if (P.counters) { P.counters[0] += nk; P.counters[1] += send - sub - nk; }
        for (int grp = 0; grp < GC::NG; grp++) group_proc<C, SR>(P, sm, grp, nk, bx, ctxs);
#endif
    }

    // ---- flush the register-resident J[ij] of the stationary bra pair
    if (P.vj && P.n_dm_j == 1) {
        B2_ALL_THREADS(tid)
            LaneCtx<C>& L = B2_CTX(tid);
            if (L.valid) {
                const int b0 = L.t.p * C::NJP;
                B2_UNROLL
                for (int bb = 0; bb < C::NJP; bb++) {
                    B2_UNROLL
                    for (int a = 0; a < C::NI; a++) {
                        double val = L.jij[bb * C::NI + a];
                        if (val != 0.0) red_add(&P.vj[(size_t)(sm.bra.i0 + a) * P.n + (sm.bra.j0 + b0 + bb)], val);
                    }
                }
            }
        B2_END
    }
#if !defined(__CUDA_ARCH__)
    delete[] ctxs;
#endif
}

}  // namespace b200jk
