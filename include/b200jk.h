/*
 * b200jk.h — C ABI of libb200jk.so, the H100-native J/K Fock-matrix builder.
 *
 * Every entry point takes plain pointers and sizes (numpy-owned host buffers); the library owns all
 * device memory, streams and NCCL communicators inside the opaque handle.  All functions return 0 on
 * success and a non-zero code on failure (message via b200jk_last_error); nothing ever calls exit().
 *
 * What each entry point replaces in the reference (file:line under /root/reference):
 *
 *   b200jk_create            the libcint tables consumed by every integral call:
 *                            Mole._atm/_bas/_env  pyscf/gto/mole.py:963-1085, slots :58-88
 *   b200jk_set_screening     _VHFOpt.__init__/init_cvhf_direct   pyscf/scf/_vhf.py:151-206
 *                            -> CVHFnr_int2e_q_cond              pyscf/lib/vhf/optimizer.c:408-454
 *   b200jk_direct_jk         _vhf.direct -> nr_direct_drv        pyscf/scf/_vhf.py:370-429,505-604
 *                            -> CVHFnr_direct_drv / CVHFdot_nrs8 pyscf/lib/vhf/nr_direct.c:361-489,183-231
 *                            -> libcint int2e_sph                (call site nr_direct.c:73)
 *                            -> nrs8_ji_s2kl / nrs8_li_s2kj      pyscf/lib/vhf/nr_direct_dot.c:1293,1435
 *                            -> CVHFnr_dm_cond, CVHFnrs8_prescreen  optimizer.c:494-518,90-117
 *                            -> lib.hermi_triu                   pyscf/lib/numpy_helper.py:499
 *   b200jk_incore_set_eri /  _vhf.incore -> CVHFnrs8_incore_drv   pyscf/scf/_vhf.py:283-366, pyscf/lib/vhf/nr_incore.c:624
 *   b200jk_incore_jk         (J/K from stored integrals, mf._eri; pyscf/scf/hf.py:2499-2508)
 *   b200jk_df_build          incore.cholesky_eri                 pyscf/df/incore.py:129-220
 *                            -> GTOnr3c_drv / GTOint2c           pyscf/lib/gto/fill_nr_3c.c:196, fill_int2c.c:36
 *   b200jk_df_prepare_j /    df_jk.get_j (integral-direct J, no tensor)  pyscf/df/df_jk.py:415-506
 *   b200jk_df_direct_j       -> CVHFnr3c2e_* passes over int3c2e  pyscf/lib/vhf/optimizer.c:305-370
 *   b200jk_df_jk             df_jk.get_jk                        pyscf/df/df_jk.py:280-413
 *                            -> AO2MOnr_e2_drv + NPdgemm         pyscf/lib/ao2mo/nr_ao2mo.c:1240, np_helper/npdot.c:32
 *   b200jk_df_ao2mo          DF.ao2mo = get_mo_eri               pyscf/df/df.py:278-296
 *                            -> _ao2mo.nr_e2 + lib.dot           pyscf/ao2mo/_ao2mo.py:157, pyscf/lib/ao2mo/nr_ao2mo.c:1240
 *   b200jk_df_get_ao_eri     DF.get_eri = get_ao_eri             pyscf/df/df.py:269-276 (+ ao2mo.restore(8))
 *   b200jk_df_mp2            DFRMP2 / DFUMP2 kernel              pyscf/mp/dfmp2.py:39-121, dfump2.py:38-166
 *                            -> MP2_contract_d, MP2_OS_contract_d pyscf/lib/mp/mp2.c:89-275
 *   b200jk_df_rpa            RPA / URPA kernel                   pyscf/gw/rpa.py:43-130, urpa.py:41-72
 *                            -> make_dielectric_matrix + log(det(I - Pi)) per frequency  rpa.py:80-84,100-130
 *   b200jk_get_stats         (no reference equivalent; logger.timer 'vj and vk' pyscf/scf/hf.py:2158)
 *
 * Conventions: all matrices are C-contiguous fp64 in the reference's spherical AO order;
 *   J_kl = sum_ij (ij|kl) D_ji ,  K_il = sum_jk (ij|kl) D_jk      (pyscf/scf/hf.py:906-907)
 * no factor 1/2, no sign.  omega: 0 full Coulomb, >0 erf(omega r12)/r12 (pyscf/gto/mole.py:2940-2951).
 */
#ifndef B200JK_H
#define B200JK_H
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

typedef struct b200jk_handle_s* b200jk_handle;

typedef struct {
    double ms_total;        /* wall time of the last J/K call inside the library (host clock) */
    double ms_kernels;      /* CUDA-event time of the J/K kernels of the last call */
    double ms_h2d, ms_d2h;  /* copies of the last call */
    uint64_t quartets_computed;  /* shell quartets that passed screening in the last direct call */
    uint64_t quartets_screened;  /* shell quartets rejected on device */
    uint64_t kernel_launches;    /* kernels launched by the last call */
    int32_t n_dev_shells, n_cart, n_sph, n_pairs;
} b200jk_stats;

/* Build a handle from libcint-layout tables (copied).  device: CUDA device ordinal. */
int b200jk_create(b200jk_handle* out, const int32_t* atm, int natm, const int32_t* bas, int nbas, const double* env,
                  int nenv, int device);
/* The same with Cartesian AOs when cart != 0 (mol.cart = True; libcint's int2e_cart, pyscf/gto/moleintor.py:772): every dm / vj /
 * vk then runs over the (l+1)(l+2)/2 Cartesian functions of each shell.  Serves the 4-center, in-core and density-fitting paths;
 * a DF tensor of such a handle is built in a Cartesian auxiliary basis (see b200jk_df_build). */
int b200jk_create2(b200jk_handle* out, const int32_t* atm, int natm, const int32_t* bas, int nbas, const double* env,
                   int nenv, int device, int cart);
int b200jk_destroy(b200jk_handle h);

/* Schwarz bounds on device + screened, sorted shell-pair lists.  Must precede b200jk_direct_jk. */
int b200jk_set_screening(b200jk_handle h, double direct_scf_tol, double omega);

/* dm: [n_dm, nao, nao]; hermi: 0 general real, 1 symmetric, 2 antisymmetric (hf.py:896-901).
 * vj / vk: [n_dm, nao, nao] outputs, either may be NULL (with_j / with_k false). */
int b200jk_direct_jk(b200jk_handle h, const double* dm, int n_dm, int nao, int hermi, double* vj, double* vk);

/* Same computation with dm and outputs already resident on the device of the handle
 * (device pointers); no host<->device copies.  Used by bench.py for the HBM-resident number. */
int b200jk_direct_jk_device(b200jk_handle h, const double* dm_dev, int n_dm, int nao, int hermi, double* vj_dev,
                            double* vk_dev);

/* In-core path: J/K from two-electron integrals the caller keeps (mf._eri): RHF.get_jk -> dot_eri_dm -> _vhf.incore ->
 * CVHFnrs8_incore_drv (pyscf/scf/hf.py:2499-2508, 902-961; pyscf/scf/_vhf.py:283-366; pyscf/lib/vhf/nr_incore.c:624).
 * eri: 8-fold packed [npair(npair+1)/2] (mol.intor('int2e', aosym='s8')), 4-fold [npair, npair] or full [nao]^4, told apart by
 * its size as dot_eri_dm does; copied to the device once.  dm: [n_dm, nao, nao] of any symmetry; vj / vk may be NULL. */
int b200jk_incore_set_eri(b200jk_handle h, const double* eri, int64_t neri, int nao);
int b200jk_incore_jk(b200jk_handle h, const double* dm, int n_dm, int nao, double* vj, double* vk);

/* Density fitting: aux tables are a second libcint-layout set for the auxiliary basis.  The auxiliary functions follow the
 * handle's AO convention, as the reference's make_auxmol copies mol.cart (pyscf/df/addons.py:245, incore.py:144-149): a
 * Cartesian handle (b200jk_create2 with cart != 0) builds cderi[naux_cart][ncart(ncart+1)/2] from int3c2e_cart / int2c2e_cart,
 * naux_cart counting (l+1)(l+2)/2 functions per auxiliary shell.  Mixing conventions is the caller's to refuse. */
int b200jk_df_build(b200jk_handle h, const int32_t* aux_atm, int aux_natm, const int32_t* aux_bas, int aux_nbas,
                    const double* aux_env, int aux_nenv, double omega, double lindep);
/* Integral-direct DF-J (df_jk.get_j, pyscf/df/df_jk.py:415-506; what DF.get_jk does for with_k=False while no tensor
 * exists, df_jk.py:282-285).  prepare_j = auxiliary tables + factorised metric (the reference's cached dfobj._vjopt);
 * direct_j = two passes over the 3-center integrals: rho = j2c^-1 (P|ij) D_ji, then J_ij = (ij|P) rho_P.  No tensor is
 * stored; b200jk_df_direct_j also works after b200jk_df_build.  dm, vj: host [n_dm, nao, nao]. */
int b200jk_df_prepare_j(b200jk_handle h, const int32_t* aux_atm, int aux_natm, const int32_t* aux_bas, int aux_nbas,
                        const double* aux_env, int aux_nenv, double omega, double lindep);
int b200jk_df_direct_j(b200jk_handle h, const double* dm, int n_dm, int nao, double* vj);
/* occ_coeff: [n_dm, nao, nocc] = C_occ*sqrt(occ) (may be NULL -> general-dm K algorithm). */
int b200jk_df_jk(b200jk_handle h, const double* dm, int n_dm, int nao, const double* occ_coeff, int nocc, int hermi,
                 double* vj, double* vk);
int b200jk_df_naux(b200jk_handle h, int* naux);
/* b200jk_df_jk with dm, occ_coeff, vj, vk already on the handle's device (device pointers, no host copies). */
int b200jk_df_jk_device(b200jk_handle h, const double* dm_dev, int n_dm, int nao, const double* occ_dev, int nocc, int hermi,
                        double* vj_dev, double* vk_dev);
/* K-build engine for the occupied-orbital path: mode 1 (default) = int8-slice tensor-core GEMMs (wgmma, i8gemm.cuh) with
 * `nslices` 7-bit slices (7 -> ~1e-11 relative), mode 0 = cuBLAS DGEMM on the FP64 pipe (kept as yardstick). */
int b200jk_df_set_kmode(b200jk_handle h, int mode, int nslices);
/* Device time of the stages of the last b200jk_df_jk[_device] call, from CUDA events recorded around every launch on
 * the launching stream (no reference equivalent; the reference brackets the whole loop with logger.timer 'vj and vk',
 * pyscf/df/df_jk.py:412): ms[s] = summed milliseconds, count[s] = launches of stage s; n <= B200JK_DF_NSTAGE entries. */
enum { B200JK_DF_STAGE_J_RHO = 0,    /* rho_P = sum cderi[P,:] dmtril           (streams the tensor once) */
       B200JK_DF_STAGE_J_ACC = 1,    /* J~ = sum_P rho_P cderi[P,:]             (streams it a second time) */
       B200JK_DF_STAGE_K_GEMM1 = 2,  /* Y = (P|mu nu) C~     i8gemm_kernel (wgmma) */
       B200JK_DF_STAGE_K_SLICE = 3,  /* int8 slicing of Y */
       B200JK_DF_STAGE_K_GEMM2 = 4,  /* K += Y Y^T           i8gemm_kernel (wgmma) */
       B200JK_DF_NSTAGE = 5 };
int b200jk_df_stage_times(b200jk_handle h, double* ms, int* count, int n);
/* Rows of the tensor held by this handle: [row0, row0+nrow) of the naux rows.  The whole tensor unless
 * b200jk_set_shard(rank, world) was called BEFORE b200jk_df_build, in which case only this rank's rows are built
 * (the 3-center integrals are computed in bounded batches of AO shell pairs and multiplied by this rank's rows of L^-1). */
int b200jk_df_local_rows(b200jk_handle h, int* row0, int* nrow);
/* Use a tensor made elsewhere instead of b200jk_df_build: cderi[naux][nao(nao+1)/2] host buffer in the reference layout
 * (mf.with_df._cderi = ndarray, pyscf/df/df.py:116, pyscf/df/test/test_df_jk.py:135-142).  Honours b200jk_set_shard (only this
 * rank's rows are uploaded).  b200jk_df_direct_j is not available on such a handle (no auxiliary basis, no metric). */
int b200jk_df_set_cderi(b200jk_handle h, const double* cderi, int naux, int nao);
/* Rows [r0, r0+nr) (LOCAL indices) of the device-resident tensor, reference layout cderi[naux, nao(nao+1)/2]
 * (pyscf/df/incore.py:134-136; what DF.loop() yields, pyscf/df/df.py:214-242). */
int b200jk_df_get_cderi(b200jk_handle h, double* out, int r0, int nr);

/* Columns cols[ncols] (packed AO-pair indices mu(mu+1)/2+nu, mu >= nu) of all LOCAL rows: out[nrow_local][ncols] — numpy
 * slicing dfobj._cderi[:, cols] on the reference's ndarray tensor (pyscf/df/df.py:116); samples a tensor too large to copy. */
int b200jk_df_get_cderi_cols(b200jk_handle h, double* out, const int64_t* cols, int ncols);

/* MO integrals from the tensor: DF.ao2mo = get_mo_eri (pyscf/df/df.py:278-296: _ao2mo.nr_e2 on each row block + lib.dot).
 * c1..c4: host [nao][n1..n4] C-contiguous coefficients over the handle's AOs (Cartesian ones on a Cartesian handle).
 * out[nij][nkl] (host) = sum_P L[P, ij] L'[P, kl], L[P, ij] = sum_{mu nu} c1[mu,i] B_P[mu,nu] c2[nu,j].  s2_12 != 0 (c1 and c2 the
 * same set, n1 == n2): ij = i(i+1)/2 + j, i >= j, nij = n1(n1+1)/2; else ij = i n2 + j.  Pair (3,4) alike; c3 == NULL: pair (3,4)
 * is pair (1,2) (the reference's sym, df.py:286-294) and only the lower output tiles are computed where a band allows it.
 * Stage 1 (half transforms, all local rows kept on the device) and stage 2 (output bands through pinned staging) run on FP64
 * tensor-core GEMMs (df_ao2mo.cuh); pair-screened tensors and host rows are read as b200jk_df_jk reads them.  Fails with a
 * message when L (and L') do not fit in device memory; a sharded tensor is refused. */
int b200jk_df_ao2mo(b200jk_handle h, const double* c1, int n1, const double* c2, int n2, int s2_12, const double* c3, int n3,
                    const double* c4, int n4, int s2_34, double* out);
/* AO integrals from the tensor: DF.get_eri = get_ao_eri (pyscf/df/df.py:269-276): ao2mo.restore(8, B^T B, nao), the lower
 * triangle row by row of the [npair, npair] matrix sum_P B[P,:]^T B[P,:] (npair = nao(nao+1)/2): out_s8[npair(npair+1)/2]. */
int b200jk_df_get_ao_eri(b200jk_handle h, double* out_s8);
/* Test hook: at most max_rows output rows per band of b200jk_df_ao2mo / b200jk_df_get_ao_eri (-1: automatic, <= 256 MiB). */
int b200jk_df_set_ao2mo_tile(b200jk_handle h, int max_rows);
/* Times of the last b200jk_df_ao2mo / b200jk_df_get_ao_eri (no reference equivalent): ms[0] stage-1 and ms[1] stage-2 device
 * time (CUDA events around the launches), ms[2] host wall time of the whole call including the copies; n <= 3 entries. */
int b200jk_df_ao2mo_times(b200jk_handle h, double* ms, int n);
/* DFMP2 / DFUMP2 kernel (pyscf/mp/dfmp2.py:39-121, dfump2.py:38-166): nspin 1 or 2; per spin s occupied / virtual
 * coefficients c_occ[s] [nao][nocc[s]] / c_vir[s] [nao][nvir[s]] (host, C-contiguous) and orbital energies e_occ[s] / e_vir[s].
 * e_out[0] = same-spin, e_out[1] = opposite-spin part of the correlation energy (e_corr = e_out[0] + e_out[1]).
 * t2: NULL, or nspin == 1: t2[0] = [nocc, nocc, nvir, nvir]; nspin == 2: t2[0..2] = aa, ab, bb as dfump2.py:51-54 (aa and bb
 * antisymmetrized as with t2_ex, mp2.c:158-161).  A spin with no occupied or no virtual orbitals contributes exactly 0.
 * (ia|jb) is formed pair by pair on the device and never leaves it (df_mp2.cuh); the energies are bit-reproducible.  Fails
 * with a message when L[naux, nocc nvir] of each spin does not fit next to the tensor; a sharded tensor is refused. */
int b200jk_df_mp2(b200jk_handle h, int nspin, const double* const* c_occ, const int* nocc, const double* const* c_vir,
                  const int* nvir, const double* const* e_occ, const double* const* e_vir, double* e_out, double* const* t2);
/* Times of the last b200jk_df_mp2: ms[0] stage-1, ms[1] stage-2 device ms, ms[2] host wall time of the call; n <= 3. */
int b200jk_df_mp2_times(b200jk_handle h, double* ms, int n);
/* Direct-RPA kernel (pyscf/gw/rpa.py:43-130, urpa.py:41-72): nspin 1 (RPA) or 2 (URPA); per spin s occupied / virtual
 * coefficients c_occ[s] [nao][nocc[s]] / c_vir[s] [nao][nvir[s]] (host, C-contiguous) and e_ov[s] / f_ov[s] [nocc[s] nvir[s]]
 * (index i nvir + a, as make_e_ov / make_f_ov return them).  For each of the nw frequencies omega[w]:
 *   Pi(w) = sum_s L_s chi_s(w) L_s^T,  chi_s[ia] = 2 e_ov f_ov / (w^2 + e_ov^2)   (make_dielectric_matrix, rpa.py:100-130)
 * logdet[w] = log det(I - Pi(w)) from a Cholesky factor and trace[w] = tr Pi(w); e_corr = sum_w weight_w / 2pi (logdet[w] +
 * trace[w]) (rpa.py:80-84).  diel: NULL, or with nw == 1, Pi(omega[0]) [naux][naux] (full and symmetric, not I - Pi).  A spin
 * with no occupied or no virtual orbitals contributes nothing.  L_s = C_occ^T B C_vir stays on the device and Pi is formed
 * there one frequency at a time (df_rpa.cuh); logdet and trace are bit-reproducible up to the factorisation.  Fails with a
 * message naming omega when I - Pi(omega) is not positive definite, when L and Pi do not fit next to the tensor, and for a
 * sharded tensor. */
int b200jk_df_rpa(b200jk_handle h, int nspin, const double* const* c_occ, const int* nocc, const double* const* c_vir,
                  const int* nvir, const double* const* e_ov, const double* const* f_ov, int nw, const double* omega,
                  double* logdet, double* trace, double* diel);
/* Times of the last b200jk_df_rpa: ms[0] stage-1, ms[1] Pi GEMM, ms[2] factorisation device ms (summed over the frequencies),
 * ms[3] host wall time of the call; n <= 4. */
int b200jk_df_rpa_times(b200jk_handle h, double* ms, int n);

/* Schwarz table q_cond[nbas,nbas] in the reference's (contracted, spherical-order) shell indexing. */
int b200jk_get_q_cond(b200jk_handle h, double* q_cond, int nbas);

/* Multi-GPU partition (one process per GPU): this handle computes only its share of the work — bra shell
 * pairs i*world+rank of every class on the 4-center path, auxiliary rows [naux*rank/world, naux*(rank+1)/world)
 * on the DF path — and returns PARTIAL J/K; the caller sums them with one all-reduce (NCCL) per build.
 * The reference analogue is the OpenMP work split + critical-section reduction, pyscf/lib/vhf/nr_direct.c:429-482. */
int b200jk_set_shard(b200jk_handle h, int rank, int world);
/* Cost table of the 4-center multi-GPU partition: measured class times ms[100] (entry [cb*10+ck], as b200jk_get_class_times
 * returns them after an UNSHARDED build with b200jk_set_profile(h, 1)).  With it every class that is small against a rank's
 * share is given whole to one rank, longest first; without it a fitted model decides and only the cheapest classes go whole.
 * All ranks must pass the same table (they derive the partition independently); NULL returns to the model. */
int b200jk_set_class_costs(b200jk_handle h, const double* ms, int n);
/* Run all work of this handle on the caller's CUDA stream (cudaStream_t cast to void*); NULL restores the
 * handle's own stream.  Lets a host framework (e.g. torch) order and time the calls with its own events. */
int b200jk_set_stream(b200jk_handle h, void* cuda_stream);
/* Register-resident DFMA micro-benchmark: measured FP64 FMA-pipe peak (TFLOP/s) of the handle's device,
 * the roofline denominator of the 4-center path (MEASURED_PEAKS.json has no fp64 entry). */
int b200jk_fp64_peak(b200jk_handle h, double* tflops);
/* Per-class kernel timing (CUDA events around each class launch; adds sync points, off by default).
 * ms[100]: entry [cb*10+ck], pair class id = l1*(l1+1)/2+l2 (ss,ps,pp,ds,dp,dd,fs,fp,fd,ff). */
int b200jk_set_profile(b200jk_handle h, int on);
int b200jk_get_class_times(b200jk_handle h, double* ms, int n);
/* Launch shape of the 4-center class (cb ck), cb >= ck (pair class ids as above), as the direct build launches it on the handle's
 * device; configures the kernel as a launch would.  info[n >= 9]: family (0 thread-per-quartet, 1 block), threads per CTA,
 * dynamic shared memory per CTA (bytes), registers per thread, local memory per thread (bytes), CTAs per SM under the carve-out
 * the library sets, that carve-out (percent, -1: none), CTAs per SM from registers and threads alone, 1 if bra and ket are
 * swapped.  Fields a CPU build cannot know are -1. */
int b200jk_class_launch_info(b200jk_handle h, int cb, int ck, int* info, int n);
/* Caps on the blocking of the int8-slice K build (tests): at most max_block_rows auxiliary rows per K block and at most
 * max_resident_rows packed rows whose slices stay resident between calls (the rest are re-cut per block); -1 keeps the
 * automatic choice, which a cap can only shrink. */
int b200jk_df_set_kblock(b200jk_handle h, int max_block_rows, int max_resident_rows);
/* Tensors larger than the device.  A handle's local rows [0, nrow) are split into device rows [0, n_dev) in HBM and host rows
 * [n_dev, nrow) in pinned host memory; every J/K call streams the host rows once through two device staging buffers (copies on a
 * copy stream of the handle, overlapped with the contraction of the previous block) and contracts J and K on each staged block.
 * The automatic split keeps every row on the device when the tensor fits next to the K workspaces; otherwise it keeps as many as
 * leave room for them and the staging buffers.  The host part is checked against MemAvailable (/proc/meminfo) first.
 * set_device_rows: cap on n_dev (-1: automatic), applied by the next b200jk_df_build / b200jk_df_set_cderi (tests, benchmarks).
 * row_split: n_dev and n_host = nrow - n_dev of the current tensor.
 * stream_stats: of the last b200jk_df_jk[_device] call: bytes copied host -> device, summed copy time and the part of it the
 * compute stream waited for (exposed_ms: copy time not hidden behind compute). */
int b200jk_df_set_device_rows(b200jk_handle h, int max_rows);
int b200jk_df_row_split(b200jk_handle h, int* n_dev, int* n_host);
int b200jk_df_stream_stats(b200jk_handle h, int64_t* bytes, double* copy_ms, double* exposed_ms);
/* Pair screening of the tensor (opt-in; the reference has no such screening).  With tol > 0 the next b200jk_df_build keeps only
 * the packed AO-pair columns (mu >= nu) whose device shell pair has a Schwarz bound q = sqrt((ab|ab)) >= tol, computed for the
 * tensor's own operator (omega) in the normalisation of b200jk_set_screening; the handle's 4-center screening state is left as
 * it is.  Dropped pairs are never integrated; device rows, pinned host rows and staging buffers hold ncol columns per row.
 * A dropped column has 2-norm <= q < tol, since ||B[:, mu nu]||^2 = (mu nu|P) M^-1 (P|mu nu) <= (mu nu|mu nu).  J of a dropped
 * pair is 0.  b200jk_df_get_cderi / _cols still return the reference layout, exact zeros at dropped columns.  tol <= 0 (the
 * default) builds the dense tensor; a tensor handed in by b200jk_df_set_cderi is always dense.
 * pair_stats: ncol kept columns of the current tensor and npair = nao(nao+1)/2. */
int b200jk_df_set_pair_tol(b200jk_handle h, double tol);
int b200jk_df_pair_stats(b200jk_handle h, int64_t* ncol, int64_t* npair);
/* Test hook: with on != 0 the next b200jk_df_build uses the identity as the metric transform (no factorisation, no
 * eigen fallback): the tensor rows are the bare 3-center integrals (P|mu nu) in the reference layout, naux = number of
 * auxiliary functions, and the assembled metric (P|Q) is kept for b200jk_df_get_metric_test.  Everything else of the build
 * (auxiliary tables, 3-center batches, transforms, pair screening, host rows, sharding) runs unchanged.  Off by default;
 * b200jk_df_direct_j refuses such a tensor. */
int b200jk_df_set_raw_test(b200jk_handle h, int on);
int b200jk_df_get_metric_test(b200jk_handle h, double* j2c, int naux);   /* [naux][naux], raw builds only */
/* Self-test of the int8-slice tensor-core GEMM used by DF-K: C[M,N] = A[M,K] B[N,K]^T with `ns` 7-bit slices (split_rows +
 * gemm_ar_acc with automatic K ranges; upper triangle only when symmetric).  b200jk_i8engine_test with stage 2. */
int b200jk_i8gemm_test(b200jk_handle h, int M, int N, int K, const double* A, const double* B, double* C, int ns,
                       int symmetric);
/* Self-test of the int8-slice engine of DF-K (i8gemm.cuh) on host buffers, `ns` 7-bit slices.  Every output may be NULL.
 * Operand A: packed = 0: a[ra][k], sliced by split_rows (the long-row kernels when k >= 8192 and ra < 4096) or, with
 *   a_rowmax[ra] (row maxima, >= 0), by split_rows_premax; packed = 1: ra packed tensor rows a[ra][k(k+1)/2] (nao = k),
 *   packed_rowexp into rowexp / rownorm2 [ra][k], then split_packed into the ra*k unpacked rows (P, a).
 * Stacks come back whole, pads included: q[ns][Rp][Kp] int8 and E[Rp] (Rp = rows rounded up to 256, Kp = k rounded up to 128).
 * stage 0: slicing only.  stage 1: b[rb][k] sliced by split_rows; gemm_ar on rows [a_row0, a_row0 + m) of A with the transposed
 *   scatter `inner` (0: none) into c ([inner][ceil(m/inner) rb], else [m][rb]) and the row maxima into rowmax ([inner] or [m],
 *   0 where none); with y_ncolp > 0 (packed A, inner = k) it writes the Y slices instead: qy / ey, Y stack of k rows and
 *   (m/k) y_ncolp columns, exponent bounds from the row norms of the block and the column norms of b.
 * stage 2: c[ra][rb] = A B^T by gemm_ar_acc from zero, upper triangle only when symmetric; kb_per > 0 forces K ranges of
 *   kb_per blocks of 128. */
typedef struct {
    int stage, packed, ns;
    const double* a; int ra, k; const double* a_rowmax;
    const double* b; int rb;
    int a_row0, m, inner, y_ncolp, symmetric, kb_per;
    int8_t* qa; int32_t* ea; int8_t* qb; int32_t* eb; int32_t* rowexp; float* rownorm2;
    double* c; double* rowmax; int8_t* qy; int32_t* ey;
} b200jk_i8test;
int b200jk_i8engine_test(b200jk_handle h, b200jk_i8test* t);
/* Self-test of the Rys quadrature of the 4-center kernels: for every x[i] (>= 0, not NaN) the n-point rule (n = 1..9) that
 * rys_root (jk_core.cuh) evaluates from the handle's device tables, in a kernel: u[count][n] roots, w[count][n] weights. */
int b200jk_rys_test(b200jk_handle h, int n, int count, const double* x, double* u, double* w);
/* Test hook of the on-device screening: the dm_cond table the last b200jk_direct_jk call screened with, dmc[nsh][nsh] over
 * the device shells (one per shell and contraction column, sorted by angular momentum; nsh = n_dev_shells of the stats), and
 * for each device shell its first AO in the caller's basis (ao_off[nsh], may be NULL): an index into the spherical AOs of
 * a b200jk_create handle, into libcint's Cartesian AOs of a b200jk_create2(..., cart = 1) handle. */
int b200jk_get_dm_cond_test(b200jk_handle h, double* dmc, int32_t* ao_off, int nsh);
int b200jk_get_stats(b200jk_handle h, b200jk_stats* out);
const char* b200jk_last_error(b200jk_handle h);
const char* b200jk_version(void);

#ifdef __cplusplus
}
#endif
#endif
